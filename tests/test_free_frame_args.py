"""CPU: gms_free_train_frame / gms_free_render_frame refuse quaternion rows that are not 16-byte aligned (the activation
kernels move them as float4) with GMS_E_ARG, before any launch."""
import ctypes as C

from gms_b200 import _lib


def _noop_alloc():
    return _lib.ALLOC_FN(lambda user, which, n: 0)


def test_misaligned_rotations_are_refused():
    L = _lib.lib()
    cb = _noop_alloc()
    base = 1 << 20          # stand-in addresses: every call below must fail its argument checks, so none is dereferenced
    a = _lib.FreeFrameArgs()
    a.P, a.M, a.scale_cols = 1, 16, 2
    a.xyz, a.scaling_raw, a.rotation_raw, a.features, a.opacity_raw = base, base, base + 4, base, base
    a.d_xyz, a.d_scaling_raw, a.d_rotation_raw, a.d_features, a.d_opacity_raw = base, base, base, base, base
    a.settings.image_width = a.settings.image_height = 16
    a.gt, a.loss, a.workspace, a.workspace_bytes = base, base, base, 0       # a too-small workspace as a second line of defence
    assert L.gms_free_train_frame(C.byref(a), cb, None, None) == _lib.GMS_E_ARG
    assert b"16-byte aligned" in L.gms_last_error()
    a.rotation_raw, a.d_rotation_raw = base, base + 8
    assert L.gms_free_train_frame(C.byref(a), cb, None, None) == _lib.GMS_E_ARG
    assert b"16-byte aligned" in L.gms_last_error()
    r = _lib.FreeRenderArgs()
    r.P, r.M, r.scale_cols = 1, 16, 3
    r.xyz, r.scaling_raw, r.rotation_raw, r.features, r.opacity_raw = base, base, base + 12, base, base
    r.settings.image_width = r.settings.image_height = 16
    r.image, r.invdepth, r.radii, r.workspace, r.workspace_bytes = base, base, base, base, 0
    assert L.gms_free_render_frame(C.byref(r), cb, None, None) == _lib.GMS_E_ARG
    assert b"16-byte aligned" in L.gms_last_error()
