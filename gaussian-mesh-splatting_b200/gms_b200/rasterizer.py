"""`diff_gaussian_rasterization`-compatible front end over libgms_b200.so.

Mirrors the Python shim of the stock extension ([upstream] diff_gaussian_rasterization/__init__.py of
graphdeco-inria/diff-gaussian-rasterization) with the API generation the reference's call sites use
(renderer/gaussian_renderer/__init__.py:43-57, 94-102): 13-field `GaussianRasterizationSettings` (incl.
`antialiasing`; a 12-field construction still works, antialiasing defaults to False) and a forward that returns
`(color [3,H,W], radii [P] int32, invdepth [1,H,W])`.

Differences that are observable only as speed: launches go to PyTorch's CURRENT stream (the stock uses the legacy
default stream), scratch memory comes from the PyTorch caching allocator through the C-ABI callback.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    antialiasing: bool = False


def _dev_f32(t: torch.Tensor, device) -> torch.Tensor:
    if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    if t.data_ptr() % 16:      # views at odd offsets: the kernels use 128-bit loads
        t = t.clone()
    return t


def _opt(t: Optional[torch.Tensor]):
    """None / empty tensor -> None (the stock shim passes torch.Tensor([]) for absent inputs)."""
    if t is None or t.numel() == 0:
        return None
    return t


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


KEEP_DEBUG = False      # tests set this to True to keep the last forward's scratch reachable
last_debug = None
last_num_rendered = 0   # N of the most recent forward (statistics for bench.py)
# When True and `shs` is a leaf whose .grad is a preallocated, zeroed, contiguous buffer (FlatAdam's contract), the
# backward kernel writes dL/dshs (192 B/Gaussian, the largest gradient) straight into it and autograd gets None:
# saves the AccumulateGrad read-modify-write over 3 x 192 MB per frame.  Off by default (plain autograd semantics).
# NOT compatible with gradient accumulation: the kernel OVERWRITES the buffer (every row, also those of culled Gaussians),
# it does not add to it -- a second backward before the optimizer step replaces the first one's SH gradient.  Callers that
# accumulate over several frames must leave this off (the default) or use one optimizer step per frame, as train.py does.
DIRECT_SH_GRAD = False


class _Scratch:
    """Holds the three scratch regions (torch uint8 tensors) alive for backward.  The ctypes callback that fills it is
    created per call and dropped right after the forward returns: keeping it would tie callback <-> owner into a
    reference cycle and leave ~300 MB per frame to the cyclic GC."""

    def __init__(self, device):
        self.device = device
        self.bufs = {}


def _make_alloc_callback(bufs: dict, device):
    def _alloc(user, which, nbytes):
        # The binning region scales with N, which changes with every camera: round it up to 64 MiB steps so the
        # caching allocator sees a handful of sizes instead of a new one per frame (a fresh cudaMalloc is a device sync).
        nbytes = int(nbytes)
        if which == _lib.BUF_BINNING:
            step = 64 << 20
            nbytes = (nbytes + step - 1) // step * step
        try:
            t = torch.empty(nbytes, dtype=torch.uint8, device=device)
        except Exception:
            return 0
        bufs[int(which)] = t
        return t.data_ptr()

    return _lib.ALLOC_FN(_alloc)


def _settings_struct(rs: GaussianRasterizationSettings, device, keep: list) -> _lib.RasterSettings:
    s = _lib.RasterSettings()
    s.image_height, s.image_width = int(rs.image_height), int(rs.image_width)
    s.tanfovx, s.tanfovy = float(rs.tanfovx), float(rs.tanfovy)
    s.scale_modifier = float(rs.scale_modifier)
    s.sh_degree = int(rs.sh_degree)
    s.prefiltered, s.debug, s.antialiasing = int(bool(rs.prefiltered)), int(bool(rs.debug)), int(bool(rs.antialiasing))
    bg, vm, pm, cp = (_dev_f32(rs.bg, device), _dev_f32(rs.viewmatrix, device), _dev_f32(rs.projmatrix, device),
                      _dev_f32(rs.campos, device))
    keep += [bg, vm, pm, cp]
    s.bg, s.viewmatrix, s.projmatrix, s.campos = bg.data_ptr(), vm.data_ptr(), pm.data_ptr(), cp.data_ptr()
    return s


def _inputs_struct(P, M, means3D, opacities, shs, colors, scales, rots, cov) -> _lib.RasterInputs:
    i = _lib.RasterInputs()
    i.P, i.M = int(P), int(M)
    i.means3D, i.opacities = _ptr(means3D), _ptr(opacities)
    i.shs, i.colors_precomp, i.scales, i.rotations, i.cov3D_precomp = _ptr(shs), _ptr(colors), _ptr(scales), _ptr(rots), _ptr(cov)
    return i


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        L = _lib.lib()
        if not means3D.is_cuda:
            raise RuntimeError("gms_b200: means3D must be a CUDA tensor (there is no CPU rasterizer in the product path)")
        device = means3D.device
        if means3D.dim() != 2 or means3D.shape[1] != 3:
            raise RuntimeError("means3D must have dimensions (num_points, 3)")
        P = means3D.shape[0]
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        f = lambda t: None if _opt(t) is None else _dev_f32(t.detach(), device)
        m3, op = _dev_f32(means3D.detach(), device), f(opacities)
        shs, col, sc, rot, cov = f(sh), f(colors_precomp), f(scales), f(rotations), f(cov3Ds_precomp)
        if P > 0 and op is None:
            raise RuntimeError("opacities must be provided")
        M = shs.shape[1] if shs is not None else 0
        keep = []
        s = _settings_struct(raster_settings, device, keep)
        i = _inputs_struct(P, M, m3, op, shs, col, sc, rot, cov)
        color = torch.empty((3, H, W), dtype=torch.float32, device=device)
        radii = torch.empty((P,), dtype=torch.int32, device=device)
        invdepth = torch.empty((1, H, W), dtype=torch.float32, device=device)
        # survivor lists for the backward pass are only worth writing when one can follow
        wants_grad = any(ctx.needs_input_grad)         # (inside Function.forward grad mode is off: ask the ctx)
        o = _lib.RasterOutputs(color.data_ptr(), radii.data_ptr(), invdepth.data_ptr(), 0 if wants_grad else _lib.FORWARD_ONLY)
        scratch = _Scratch(device)
        saved = _lib.RasterSaved()
        stream = torch.cuda.current_stream(device).cuda_stream
        cb = _make_alloc_callback(scratch.bufs, device)
        with torch.cuda.device(device):
            rc = L.gms_rasterize_forward(C.byref(s), C.byref(i), C.byref(o), cb, None, C.byref(saved), stream)
        del cb
        if rc != 0 and raster_settings.debug:
            try:
                torch.save(tuple(t.cpu() if isinstance(t, torch.Tensor) else t for t in
                                 (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)), "snapshot_fw.dump")
                print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
            except Exception:
                pass
        _lib.check(rc, "gms_rasterize_forward")
        global last_num_rendered
        last_num_rendered = int(saved.num_rendered)
        if KEEP_DEBUG:
            global last_debug
            last_debug = dict(scratch=scratch, num_rendered=int(saved.num_rendered), P=P, W=W, H=H, radii=radii,
                              bin_state=(int(saved.binning_capacity), int(saved.flags)))
        ctx.sh_sink = None
        if DIRECT_SH_GRAD and sh is not None and shs is not None and sh.is_leaf and sh.grad is not None and \
                sh.grad.is_contiguous() and sh.grad.shape == shs.shape and sh.grad.dtype == torch.float32 and \
                sh.grad.data_ptr() % 16 == 0 and sh.data_ptr() == shs.data_ptr():
            ctx.sh_sink = sh.grad
        ctx.raster_settings = raster_settings
        ctx.num_rendered = int(saved.num_rendered)
        ctx.bin_state = (int(saved.binning_capacity), int(saved.flags))
        ctx.scratch = scratch
        ctx.keep = keep
        ctx.dims = (P, M)
        ctx.present = (shs is not None, col is not None, sc is not None, rot is not None, cov is not None)
        ctx.save_for_backward(m3, op if op is not None else torch.empty(0, device=device), shs, col, sc, rot, cov, radii)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)     # an unused inverse-depth output arrives as None -> depth channel compiled out
        return color, radii, invdepth

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii, grad_out_depth):
        L = _lib.lib()
        m3, op, shs, col, sc, rot, cov, radii = ctx.saved_tensors
        device = m3.device
        P, M = ctx.dims
        rs = ctx.raster_settings
        keep = []
        s = _settings_struct(rs, device, keep)
        i = _inputs_struct(P, M, m3, op if op.numel() else None, shs, col, sc, rot, cov)
        saved = _lib.RasterSaved()
        b = ctx.scratch.bufs
        saved.geom = _ptr(b.get(_lib.BUF_GEOM)); saved.binning = _ptr(b.get(_lib.BUF_BINNING)); saved.image = _ptr(b.get(_lib.BUF_IMAGE))
        saved.num_rendered = ctx.num_rendered
        saved.binning_capacity, saved.flags = ctx.bin_state
        if grad_out_color is None:
            grad_out_color = torch.zeros((3, int(rs.image_height), int(rs.image_width)), dtype=torch.float32, device=device)
        gcol = _dev_f32(grad_out_color, device)
        gdep = None if grad_out_depth is None else _dev_f32(grad_out_depth, device)
        e = lambda *shape: torch.empty(shape, dtype=torch.float32, device=device)
        g_m3, g_m2, g_op = e(P, 3), e(P, 3), e(P, 1)
        sink = ctx.sh_sink
        g_sh = (sink if sink is not None else e(P, M, 3)) if shs is not None else None
        g_col = e(P, 3) if col is not None else None
        g_sc = e(P, 3) if sc is not None else None
        g_rot = e(P, 4) if rot is not None else None
        g_cov = e(P, 6) if cov is not None else None
        gr = _lib.RasterGrads(_ptr(g_m3), _ptr(g_m2), _ptr(g_op), _ptr(g_sh), _ptr(g_col), _ptr(g_sc), _ptr(g_rot), _ptr(g_cov))
        stream = torch.cuda.current_stream(device).cuda_stream
        with torch.cuda.device(device):
            rc = L.gms_rasterize_backward(C.byref(s), C.byref(i), radii.data_ptr(), C.byref(saved), gcol.data_ptr(),
                                          _ptr(gdep), C.byref(gr), stream)
        if rc != 0 and rs.debug:
            try:
                torch.save((m3.cpu(), radii.cpu(), gcol.cpu()), "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
            except Exception:
                pass
        _lib.check(rc, "gms_rasterize_backward")
        if P == 0:
            z = lambda t: None if t is None else torch.zeros_like(t)
            g_m3, g_m2, g_op, g_sh, g_col, g_sc, g_rot, g_cov = map(z, (g_m3, g_m2, g_op, g_sh, g_col, g_sc, g_rot, g_cov))
        if sink is not None:
            g_sh = None      # already written in place
        return g_m3, g_m2, g_sh, g_col, g_op, g_sc, g_rot, g_cov, None


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                     raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            rs = self.raster_settings
            device = positions.device
            pos = _dev_f32(positions, device)
            vm, pm = _dev_f32(rs.viewmatrix, device), _dev_f32(rs.projmatrix, device)
            present = torch.empty((pos.shape[0],), dtype=torch.bool, device=device)
            rc = _lib.lib().gms_mark_visible(pos.shape[0], pos.data_ptr(), vm.data_ptr(), pm.data_ptr(),
                                             present.data_ptr(), torch.cuda.current_stream(device).cuda_stream)
            _lib.check(rc, "gms_mark_visible")
        return present

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, rs)


def forward_debug_state(ctx_scratch: _Scratch, num_rendered: int, P: int, W: int, H: int, radii: torch.Tensor, bin_state=None):
    """Parity-test helper: unpack the library's intermediate buffers into torch tensors (stock layouts).
    bin_state = (binning_capacity, flags) of the forward call (default: taken from last_debug)."""
    if bin_state is None:
        bin_state = (last_debug or {}).get("bin_state", (0, 0))
    L = _lib.lib()
    device = radii.device
    saved = _lib.RasterSaved()
    b = ctx_scratch.bufs
    saved.geom = _ptr(b.get(_lib.BUF_GEOM)); saved.binning = _ptr(b.get(_lib.BUF_BINNING)); saved.image = _ptr(b.get(_lib.BUF_IMAGE))
    saved.num_rendered = int(num_rendered)
    saved.binning_capacity, saved.flags = int(bin_state[0]), int(bin_state[1])
    out = {}
    if P > 0:
        means2D = torch.zeros(P, 2, device=device); depths = torch.zeros(P, device=device)
        conic = torch.zeros(P, 4, device=device); rgb = torch.zeros(P, 3, device=device)
        cl = torch.zeros(P, 3, dtype=torch.uint8, device=device)
        rc = L.gms_debug_unpack(C.byref(saved), P, radii.data_ptr(), means2D.data_ptr(), depths.data_ptr(), conic.data_ptr(),
                                rgb.data_ptr(), cl.data_ptr(), torch.cuda.current_stream(device).cuda_stream)
        _lib.check(rc, "gms_debug_unpack")
        out.update(means2D=means2D, depths=depths, conic_opacity=conic, rgb=rgb, clamped=cl)
    v = _lib.DebugViews()
    _lib.check(L.gms_debug_get_views(C.byref(saved), P, W, H, C.byref(v)), "gms_debug_get_views")
    T = ((W + 15) // 16) * ((H + 15) // 16)

    def view(ptr, n, dtype):
        if not ptr or n == 0:
            return torch.zeros(0, dtype=dtype, device=device)
        nbytes = n * torch.empty(0, dtype=dtype).element_size()
        for t in b.values():   # locate the owning scratch tensor and slice it
            base = t.data_ptr()
            if base <= ptr < base + t.numel():
                return t[ptr - base: ptr - base + nbytes].view(dtype).clone()
        raise RuntimeError("debug view outside scratch")

    if P > 0:
        out["cov3D"] = view(v.cov3D, 6 * P, torch.float32).view(P, 6)
        out["tiles_touched"] = view(v.tiles_touched, P, torch.int32)
    out["point_list"] = view(v.point_list, int(num_rendered), torch.int32)
    out["ranges"] = view(v.ranges, 2 * T, torch.int32).view(T, 2)
    if v.tile_keys:
        out["tile_keys"] = view(v.tile_keys, int(num_rendered), torch.int32)
    else:   # counting binning materialises no key array: the tile of every list position follows from the ranges
        cnt = (out["ranges"][:, 1] - out["ranges"][:, 0]).long()
        start = out["ranges"][:, 0].long()
        tk = torch.full((int(num_rendered),), -1, dtype=torch.int32, device=device)
        tiles_ne = torch.nonzero(cnt > 0).flatten()
        if tiles_ne.numel():
            c = cnt[tiles_ne]
            pos = torch.repeat_interleave(start[tiles_ne], c) + \
                (torch.arange(int(c.sum()), device=device) - torch.repeat_interleave(torch.cumsum(c, 0) - c, c))
            tk[pos] = torch.repeat_interleave(tiles_ne, c).int()
        out["tile_keys"] = tk
    if v.dgeom and P > 0:
        out["dgeom"] = view(v.dgeom, 12 * P, torch.float32).view(P, 12)     # meaningful after a backward call
    out["final_T"] = view(v.final_T, W * H, torch.float32).view(H, W)
    out["n_contrib"] = view(v.n_contrib, W * H, torch.int32).view(H, W)
    if v.surv and v.nsurv:      # the forward wrote per-quad survivor lists (flags bit 1): quad q of tile t at 4 * start + q * len
        out["surv"] = view(v.surv, 4 * int(num_rendered), torch.int32)
        out["nsurv"] = view(v.nsurv, 4 * T, torch.int32).view(T, 4)
    return out
