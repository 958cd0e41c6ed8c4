"""ctypes front-end of the C oracle (oracle/gms_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of gms_oracle.c.  Parity status of the
rasterizer oracle: "parity unpinned" by reference tests (the reference has none and
the rasterizer source is an un-vendored submodule); pinned instead by golden vectors
made from the reference's own Python restatements (tests/golden/) and by the dense
autograd model in oracle/torch_dense.py.

The functions here take/return numpy arrays (float32 / int32 / uint8).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgms_oracle.so")
_lib = None

BLOCK = 16


class GmsoSettings(ctypes.Structure):
    _fields_ = [
        ("P", ctypes.c_int32), ("D", ctypes.c_int32), ("M", ctypes.c_int32),
        ("W", ctypes.c_int32), ("H", ctypes.c_int32),
        ("tanfovx", ctypes.c_float), ("tanfovy", ctypes.c_float),
        ("scale_modifier", ctypes.c_float),
        ("prefiltered", ctypes.c_int32), ("antialiasing", ctypes.c_int32),
        ("viewmatrix", ctypes.c_float * 16), ("projmatrix", ctypes.c_float * 16),
        ("campos", ctypes.c_float * 3), ("bg", ctypes.c_float * 3),
    ]


def build(force: bool = False) -> str:
    """Compile the oracle with the recipe in oracle/Makefile."""
    src = os.path.join(_HERE, "gms_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B"])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.gmso_bin.restype = ctypes.c_int64
        _lib.gmso_num_threads.restype = ctypes.c_int
        _lib.gmso_f2i_sat.restype = ctypes.c_int32
        _lib.gmso_f2i_sat.argtypes = [ctypes.c_float]
    return _lib


def f2i_sat(v: float) -> int:
    """The oracle's float -> int32 conversion (device cvt.rzi.s32.f32 semantics: saturating, NaN -> 0)."""
    return int(lib().gmso_f2i_sat(float(v)))


def num_threads() -> int:
    return int(lib().gmso_num_threads())


def set_num_threads(n: int) -> None:
    lib().gmso_set_num_threads(int(n))


def set_tile_stride(stride: int) -> None:
    """Composite only every `stride`-th tile (bounded CPU-baseline samples); 1 = all tiles."""
    lib().gmso_set_tile_stride(int(stride))


def _p(a: Optional[np.ndarray]):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "oracle arrays must be contiguous"
    return a.ctypes.data_as(ctypes.c_void_p)


def _f32(a):
    if a is None:
        return None
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


@dataclass
class Settings:
    """Mirror of GaussianRasterizationSettings (renderer/gaussian_renderer/__init__.py:43-57)."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: np.ndarray
    scale_modifier: float
    viewmatrix: np.ndarray   # [4,4] world_view_transform (transposed W2C)
    projmatrix: np.ndarray   # [4,4] full_proj_transform
    sh_degree: int
    campos: np.ndarray
    prefiltered: bool = False
    debug: bool = False
    antialiasing: bool = False

    def to_c(self, P: int, M: int) -> GmsoSettings:
        s = GmsoSettings()
        s.P, s.D, s.M = int(P), int(self.sh_degree), int(M)
        s.W, s.H = int(self.image_width), int(self.image_height)
        s.tanfovx, s.tanfovy = float(self.tanfovx), float(self.tanfovy)
        s.scale_modifier = float(self.scale_modifier)
        s.prefiltered, s.antialiasing = int(self.prefiltered), int(self.antialiasing)
        vm = _f32(self.viewmatrix).reshape(16)
        pm = _f32(self.projmatrix).reshape(16)
        for k in range(16):
            s.viewmatrix[k] = float(vm[k])
            s.projmatrix[k] = float(pm[k])
        cp = _f32(self.campos).reshape(3)
        bg = _f32(self.bg).reshape(3)
        for k in range(3):
            s.campos[k] = float(cp[k])
            s.bg[k] = float(bg[k])
        return s


@dataclass
class ForwardState:
    settings: Settings
    cs: GmsoSettings
    inputs: dict
    radii: np.ndarray
    means2D: np.ndarray
    depths: np.ndarray
    cov3Ds: np.ndarray
    conic_opacity: np.ndarray
    rgb: np.ndarray
    clamped: np.ndarray
    tiles_touched: np.ndarray
    rects: np.ndarray
    offsets: np.ndarray = None
    N: int = 0
    keys_sorted: np.ndarray = None
    point_list: np.ndarray = None
    ranges: np.ndarray = None
    color: np.ndarray = None
    final_T: np.ndarray = None
    n_contrib: np.ndarray = None
    invdepth: np.ndarray = None
    ambiguous: np.ndarray = None
    extra: dict = field(default_factory=dict)


def preprocess(settings: Settings, means3D, opacities, shs=None, colors_precomp=None,
               scales=None, rotations=None, cov3D_precomp=None) -> ForwardState:
    means3D = _f32(means3D).reshape(-1, 3)
    P = means3D.shape[0]
    opacities = _f32(opacities).reshape(-1)
    shs = _f32(shs)
    colors_precomp = _f32(colors_precomp)
    scales = _f32(scales)
    rotations = _f32(rotations)
    cov3D_precomp = _f32(cov3D_precomp)
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    M = shs.shape[1] if shs is not None else 0
    cs = settings.to_c(P, M)
    radii = np.zeros(P, np.int32)
    means2D = np.zeros((P, 2), np.float32)
    depths = np.zeros(P, np.float32)
    cov3Ds = np.zeros((P, 6), np.float32)
    conic_opacity = np.zeros((P, 4), np.float32)
    rgb = np.zeros((P, 3), np.float32)
    clamped = np.zeros((P, 3), np.uint8)
    tiles = np.zeros(P, np.uint32)
    rects = np.zeros((P, 4), np.int32)
    rc = lib().gmso_preprocess_forward(ctypes.byref(cs), _p(means3D), _p(scales), _p(rotations),
                                       _p(cov3D_precomp), _p(opacities), _p(shs), _p(colors_precomp),
                                       _p(radii), _p(means2D), _p(depths), _p(cov3Ds), _p(conic_opacity),
                                       _p(rgb), _p(clamped), _p(tiles), _p(rects))
    if rc != 0:
        raise RuntimeError(f"gmso_preprocess_forward failed rc={rc}")
    inputs = dict(means3D=means3D, opacities=opacities, shs=shs, colors_precomp=colors_precomp,
                  scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
    return ForwardState(settings, cs, inputs, radii, means2D, depths, cov3Ds, conic_opacity, rgb,
                        clamped, tiles, rects)


def bin_tiles(st: ForwardState) -> ForwardState:
    P = st.radii.shape[0]
    W, H = st.settings.image_width, st.settings.image_height
    T = ((W + BLOCK - 1) // BLOCK) * ((H + BLOCK - 1) // BLOCK)
    st.offsets = np.zeros(P, np.uint32)
    N = int(st.tiles_touched.astype(np.int64).sum())
    st.keys_sorted = np.zeros(max(N, 1), np.uint64)
    st.point_list = np.zeros(max(N, 1), np.uint32)
    st.ranges = np.zeros((T, 2), np.int32)
    n = lib().gmso_bin(ctypes.byref(st.cs), _p(st.radii), _p(st.depths), _p(st.rects),
                       _p(st.tiles_touched), _p(st.offsets), _p(st.keys_sorted), _p(st.point_list),
                       _p(st.ranges), ctypes.c_int64(max(N, 1)))
    assert n == N, (n, N)
    st.N = N
    st.keys_sorted = st.keys_sorted[:N]
    st.point_list = st.point_list[:N]
    return st


def composite(st: ForwardState) -> ForwardState:
    W, H = st.settings.image_width, st.settings.image_height
    st.color = np.zeros((3, H, W), np.float32)
    st.final_T = np.zeros((H, W), np.float32)
    st.n_contrib = np.zeros((H, W), np.int32)
    st.invdepth = np.zeros((1, H, W), np.float32)
    st.ambiguous = np.zeros((H, W), np.uint8)
    pl = st.point_list if st.N > 0 else np.zeros(1, np.uint32)
    lib().gmso_composite_forward(ctypes.byref(st.cs), _p(st.ranges), _p(pl), _p(st.means2D),
                                 _p(st.rgb), _p(st.conic_opacity), _p(st.depths), _p(st.color),
                                 _p(st.final_T), _p(st.n_contrib), _p(st.invdepth), _p(st.ambiguous))
    return st


def forward(settings: Settings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
            rotations=None, cov3D_precomp=None) -> ForwardState:
    """Whole forward pass: returns the state with color [3,H,W], radii [P], invdepth [1,H,W]."""
    st = preprocess(settings, means3D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp)
    bin_tiles(st)
    composite(st)
    return st


def composite_backward(st: ForwardState, dL_dcolor, dL_dinvdepth=None) -> dict:
    P = st.radii.shape[0]
    dL_dcolor = _f32(dL_dcolor).reshape(3, st.settings.image_height, st.settings.image_width)
    dinv = _f32(dL_dinvdepth)
    if dinv is not None:
        dinv = dinv.reshape(st.settings.image_height, st.settings.image_width)
    g = dict(dL_dmean2D=np.zeros((P, 2), np.float64), dL_dconic=np.zeros((P, 3), np.float64),
             dL_dopacity=np.zeros(P, np.float64), dL_dcolor=np.zeros((P, 3), np.float64),
             dL_dinvdepth=np.zeros(P, np.float64))
    pl = st.point_list if st.N > 0 else np.zeros(1, np.uint32)
    lib().gmso_composite_backward(ctypes.byref(st.cs), _p(st.ranges), _p(pl), _p(st.means2D), _p(st.rgb),
                                  _p(st.conic_opacity), _p(st.depths), _p(st.final_T), _p(st.n_contrib),
                                  _p(dL_dcolor), _p(dinv), _p(g["dL_dmean2D"]), _p(g["dL_dconic"]),
                                  _p(g["dL_dopacity"]), _p(g["dL_dcolor"]), _p(g["dL_dinvdepth"]))
    return g


def composite_backward64(st: ForwardState, dL_dcolor, dL_dinvdepth=None) -> dict:
    """The composite backward evaluated in float64 on the fp32 forward's blend decisions, with a per-element error budget
    (gmso_composite_backward64 in gms_oracle.c derives it).  Returns ref64 [P,10] and budget [P,10] in the order of the
    kernels' per-Gaussian record (mean2D x/y, conic xx/xy/yy, opacity, rgb, inverse depth) and amb_share [P]: the largest
    share of a Gaussian's budget that comes from the allowance at threshold-ambiguous pixels."""
    P = st.radii.shape[0]
    H, W = st.settings.image_height, st.settings.image_width
    dL_dcolor = _f32(dL_dcolor).reshape(3, H, W)
    dinv = _f32(dL_dinvdepth)
    if dinv is not None:
        dinv = dinv.reshape(H, W)
    out = dict(ref64=np.zeros((P, 10), np.float64), budget=np.zeros((P, 10), np.float64), amb_share=np.zeros(P, np.float64))
    pl = st.point_list if st.N > 0 else np.zeros(1, np.uint32)
    amb = np.ascontiguousarray(st.ambiguous, dtype=np.uint8)
    rc = lib().gmso_composite_backward64(ctypes.byref(st.cs), _p(st.ranges), _p(pl), _p(st.means2D), _p(st.rgb),
                                         _p(st.conic_opacity), _p(st.depths), _p(st.n_contrib), _p(amb), _p(dL_dcolor),
                                         _p(dinv), _p(out["ref64"]), _p(out["budget"]), _p(out["amb_share"]))
    if rc != 0:
        raise RuntimeError(f"gmso_composite_backward64 failed rc={rc}")
    return out


FWD64_OUTPUTS = ("r", "g", "b", "invdepth", "final_T")


def composite_forward64(st: ForwardState, rgb=None, rgb_tol: float = 0.0) -> dict:
    """The composite forward evaluated in float64 on the fp32 forward's blend decisions, with a per-pixel error budget
    (gmso_composite_forward64 in gms_oracle.c derives it).  Returns ref [5,H,W] and budget [5,H,W] (colour r/g/b, inverse
    depth, final T), allowance [5,H,W] (the share of the budget from flip candidates), adm [H,W,8] (admissible n_contrib;
    -1 pads, -2 admits any value >= adm[..., 0]), cand [H,W] (pixels with a flip candidate), qhit [N] and qcand [N] (per list
    position, bit q: the splat blends at / may flip at some pixel of quad q of its tile).  `rgb` [P,3] replaces the oracle's
    colours (the kernels' own record); `rgb_tol` widens the budget for a colour record known only to that tolerance."""
    H, W = st.settings.image_height, st.settings.image_width
    rgb = st.rgb if rgb is None else np.ascontiguousarray(rgb, dtype=np.float32).reshape(st.rgb.shape)
    n = max(st.N, 1)
    out = dict(ref=np.zeros((5, H, W)), budget=np.zeros((5, H, W)), allowance=np.zeros((5, H, W)),
               adm=np.zeros((H, W, 8), np.int32), cand=np.zeros((H, W), np.uint8), qhit=np.zeros(n, np.uint8),
               qcand=np.zeros(n, np.uint8))
    pl = st.point_list if st.N > 0 else np.zeros(1, np.uint32)
    rc = lib().gmso_composite_forward64(ctypes.byref(st.cs), _p(st.ranges), _p(pl), _p(st.means2D), _p(rgb),
                                        _p(st.conic_opacity), _p(st.depths), ctypes.c_double(rgb_tol), _p(out["ref"]),
                                        _p(out["budget"]), _p(out["allowance"]), _p(out["adm"]), _p(out["cand"]),
                                        _p(out["qhit"]), _p(out["qcand"]))
    if rc != 0:
        raise RuntimeError(f"gmso_composite_forward64 failed rc={rc}")
    out["qhit"], out["qcand"] = out["qhit"][:st.N], out["qcand"][:st.N]
    return out


def preprocess_backward(st: ForwardState, g: dict) -> dict:
    P = st.radii.shape[0]
    inp = st.inputs
    M = st.cs.M
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    d2 = f(g["dL_dmean2D"]); dcon = f(g["dL_dconic"]); dop = f(g["dL_dopacity"])
    dcol = f(g["dL_dcolor"]); dinv = f(g["dL_dinvdepth"])
    out = dict(dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dcov3D=np.zeros((P, 6), np.float32),
               dL_dopacity=np.zeros((P, 1), np.float32))
    dsh = np.zeros((P, M, 3), np.float32) if inp["shs"] is not None else None
    dcp = np.zeros((P, 3), np.float32) if inp["colors_precomp"] is not None else None
    dsc = np.zeros((P, 3), np.float32) if inp["scales"] is not None else None
    drot = np.zeros((P, 4), np.float32) if inp["rotations"] is not None else None
    lib().gmso_preprocess_backward(ctypes.byref(st.cs), _p(st.radii), _p(inp["means3D"]), _p(inp["scales"]),
                                   _p(inp["rotations"]), _p(inp["cov3D_precomp"]), _p(inp["opacities"]),
                                   _p(inp["shs"]), _p(inp["colors_precomp"]), _p(st.cov3Ds), _p(st.clamped),
                                   _p(d2), _p(dcon), _p(dop), _p(dcol), _p(dinv),
                                   _p(out["dL_dmeans3D"]), _p(out["dL_dcov3D"]), _p(dsh), _p(dcp), _p(dsc),
                                   _p(drot), _p(out["dL_dopacity"]))
    out["dL_dmeans2D"] = np.concatenate([d2, np.zeros((P, 1), np.float32)], axis=1)
    out["dL_dsh"] = dsh
    out["dL_dcolors_precomp"] = dcp
    out["dL_dscales"] = dsc
    out["dL_drotations"] = drot
    return out


def backward(st: ForwardState, dL_dcolor, dL_dinvdepth=None) -> dict:
    """Whole backward pass; returns gradients keyed like the autograd outputs of the rasterizer."""
    g = composite_backward(st, dL_dcolor, dL_dinvdepth)
    out = preprocess_backward(st, g)
    out["_composite"] = g
    # the upstream gradients, for checks that re-evaluate the composite backward (composite_backward64)
    out["_upstream"] = (dL_dcolor, dL_dinvdepth)
    return out


def mark_visible(settings: Settings, means3D) -> np.ndarray:
    means3D = _f32(means3D).reshape(-1, 3)
    cs = settings.to_c(means3D.shape[0], 0)
    present = np.zeros(means3D.shape[0], np.uint8)
    lib().gmso_mark_visible(ctypes.byref(cs), _p(means3D), _p(present))
    return present.astype(bool)
