"""CPU: the seven one-call frame entry points refuse malformed arguments with GMS_E_ARG and a fixed message, in a fixed
order of checks, before any CUDA call; and the frame / render workspace sizes and the frame-view offsets stay put.

Every case starts from arguments that pass every check but the last one (the workspace is one byte short), so no call
below can reach a launch.  Cases with two faults pin which check runs first."""
import ctypes as C

import pytest

from gms_b200 import _lib

BASE = 1 << 20      # stand-in device address, 16-byte aligned: every call fails its argument checks, so none is dereferenced
P_FREE, F_MESH, K_MESH = 6, 3, 2


def _settings(s):
    s.image_width, s.image_height, s.sh_degree = 16, 16, 3
    s.bg = s.viewmatrix = s.projmatrix = s.campos = BASE


def _render_outputs(a, ws_bytes):
    a.image = a.invdepth = a.radii = BASE
    a.workspace, a.workspace_bytes = BASE, ws_bytes - 1


def _mesh_model(a):
    a.V, a.F, a.K, a.M = 4, F_MESH, K_MESH, 16
    a.vertices = a.faces = a.alpha_raw = a.scale_raw = a.features = a.opacity_raw = BASE
    a.alpha_activation = _lib.ALPHA_RELU


def _free_model(a):
    a.P, a.M, a.scale_cols = P_FREE, 16, 3
    a.xyz = a.scaling_raw = a.rotation_raw = a.features = a.opacity_raw = BASE


def _render():
    a = _lib.RenderArgs()
    _mesh_model(a)
    _settings(a.settings)
    _render_outputs(a, _lib.lib().gms_render_workspace_bytes(F_MESH * K_MESH, 16, 16))
    return a


def _points_render():
    a = _lib.PointsRenderArgs()
    a.P, a.M = P_FREE, 16
    a.triangles = a.features = a.opacity_raw = BASE
    _settings(a.settings)
    _render_outputs(a, _lib.lib().gms_points_render_workspace_bytes(P_FREE, 16, 16))
    return a


def _bound_points_render():
    a = _lib.BoundPointsRenderArgs()
    a.P, a.M, a.V, a.F = P_FREE, 16, 4, 2
    a.face = a.coeffs = a.vertices = a.faces = a.features = a.opacity_raw = BASE
    _settings(a.settings)
    _render_outputs(a, _lib.lib().gms_bound_points_render_workspace_bytes(P_FREE, 16, 16))
    return a


def _free_render():
    a = _lib.FreeRenderArgs()
    _free_model(a)
    _settings(a.settings)
    _render_outputs(a, _lib.lib().gms_render_workspace_bytes(P_FREE, 16, 16))
    return a


def _flame_render():
    a = _lib.FlameRenderArgs()
    a.V, a.F, a.K, a.M = 4, F_MESH, K_MESH, 16
    a.vertices = a.faces = a.alpha = a.scaling_log = a.rotation_raw = a.features = a.opacity_raw = BASE
    _settings(a.settings)
    _render_outputs(a, _lib.lib().gms_flame_render_workspace_bytes(F_MESH * K_MESH, 16, 16))
    return a


def _train():
    a = _lib.FrameArgs()
    _mesh_model(a)
    a.d_vertices = a.d_alpha_raw = a.d_scale_raw = a.d_features = a.d_opacity_raw = BASE
    _settings(a.settings)
    a.gt = a.loss = a.workspace = BASE
    a.workspace_bytes = _lib.lib().gms_frame_workspace_bytes(F_MESH * K_MESH, 16, 16) - 1
    return a


def _free_train():
    a = _lib.FreeFrameArgs()
    _free_model(a)
    a.d_xyz = a.d_scaling_raw = a.d_rotation_raw = a.d_features = a.d_opacity_raw = BASE
    _settings(a.settings)
    a.gt = a.loss = a.workspace = BASE
    a.workspace_bytes = _lib.lib().gms_frame_workspace_bytes(P_FREE, 16, 16) - 1
    return a


ENTRIES = {"gms_render_frame": _render, "gms_points_render_frame": _points_render,
           "gms_bound_points_render_frame": _bound_points_render, "gms_free_render_frame": _free_render,
           "gms_flame_render_frame": _flame_render, "gms_train_frame": _train, "gms_free_train_frame": _free_train}


def _segments(a, segs):
    arr = _lib.mesh_segments(segs)
    a.segments, a.n_segments = C.cast(arr, C.POINTER(_lib.MeshSegment)), len(segs)
    return arr


def _sh_adam(a, m=BASE, v=BASE, step=1):
    s = _lib.ShAdam()
    s.m, s.v, s.step = m, v, step
    a.sh_adam = C.pointer(s)
    return s


def _set(**fields):
    def f(a):
        for k, v in fields.items():
            assert k in dict(type(a)._fields_), k
            setattr(a, k, v)
    return f


def _set_settings(**fields):
    def f(a):
        for k, v in fields.items():
            setattr(a.settings, k, v)
    return f


def _both(*fs):
    def f(a):
        return [g(a) for g in fs]
    return f


NULL = "null argument"
WS = "workspace too small"
MESH_MODEL = "model tensors required"
MESH_GRADS = "gradient tensors required"
SEG_NULL = "n_segments < 0, or segments NULL with n_segments > 0"
SEG_K = "K must be 0 when segments are given"
SEG_FK = "every segment needs F >= 1 and K >= 1"
SEG_F = "F must equal the sum of the segments' F"
SEG_SUM = "sum of F_i * K_i over the segments exceeds int32"
ALPHA = "alpha_activation must be 0 (relu) or 1 (softmax)"
FREE_MODEL = "need P >= 0, 1 <= M <= 16, scale_cols 2 or 3 and every model tensor"
FLAME_SIZES = "need F >= 0, K >= 1, V >= 1, 1 <= M <= 16 and F*K < 2^31"
BOUND_SIZES = "need P >= 0, F >= 1, V >= 1"

# (case id, mutation, the message after "<entry>: "); the mutation "alloc" passes a NULL allocator, "args" NULL arguments
_mesh_cases = [
    ("no_alloc", "alloc", NULL), ("workspace", _set(workspace=None), NULL), ("vertices", _set(vertices=None), MESH_MODEL),
    ("faces", _set(faces=None), MESH_MODEL), ("alpha_raw", _set(alpha_raw=None), MESH_MODEL),
    ("scale_raw", _set(scale_raw=None), MESH_MODEL), ("features", _set(features=None), MESH_MODEL),
    ("opacity_raw", _set(opacity_raw=None), MESH_MODEL),
    ("alpha_activation", _set(alpha_activation=2), ALPHA), ("alpha_activation_neg", _set(alpha_activation=-1), ALPHA),
    ("n_segments_neg", _set(n_segments=-1), SEG_NULL), ("segments_null", _set(n_segments=2), SEG_NULL),
    ("segments_with_K", lambda a: _segments(a, [(1, 2), (2, 3)]), SEG_K),
    ("segment_F0", lambda a: (_segments(a, [(0, 2), (3, 3)]), setattr(a, "K", 0)), SEG_FK),
    ("segment_K0", lambda a: (_segments(a, [(1, 2), (2, 0)]), setattr(a, "K", 0)), SEG_FK),
    ("segments_F_mismatch", lambda a: (_segments(a, [(1, 2), (1, 3)]), setattr(a, "K", 0)), SEG_F),
    ("segments_overflow", lambda a: (_segments(a, [(1, 1 << 30), (2, 1 << 30)]), setattr(a, "K", 0)), SEG_SUM),
    ("segments_ok", lambda a: (_segments(a, [(1, 2), (2, 2)]), setattr(a, "K", 0)), WS),
    ("F_neg", _set(F=-1), WS),
    ("workspace_short", _set(), WS),
    # two faults: the first check wins
    ("vertices_and_alpha", _both(_set(vertices=None), _set(alpha_activation=5)), MESH_MODEL),
    ("alpha_and_segments", _both(_set(alpha_activation=5), _set(n_segments=-1)), ALPHA),
    ("segments_F_and_sum", lambda a: (_segments(a, [(1, 1 << 30), (1, 1 << 30)]), setattr(a, "K", 0)), SEG_F),
    ("segments_K_and_F0", lambda a: _segments(a, [(0, 2), (3, 3)]), SEG_K),
    ("workspace_and_model", _both(_set(workspace=None), _set(features=None)), NULL),
]

CASES = []
for _entry in ("gms_render_frame", "gms_train_frame"):
    CASES += [(_entry,) + c for c in _mesh_cases]
for _entry in ("gms_render_frame", "gms_points_render_frame", "gms_bound_points_render_frame", "gms_free_render_frame",
               "gms_flame_render_frame"):
    CASES += [(_entry, "image", _set(image=None), NULL), (_entry, "invdepth", _set(invdepth=None), NULL),
              (_entry, "radii", _set(radii=None), NULL), (_entry, "args", "args", NULL),
              (_entry, "radii_and_workspace", _both(_set(radii=None), _set(workspace_bytes=0)), NULL)]
CASES += [
    ("gms_points_render_frame", "no_alloc", "alloc", NULL),
    ("gms_points_render_frame", "triangles", _set(triangles=None), MESH_MODEL),
    ("gms_points_render_frame", "features", _set(features=None), MESH_MODEL),
    ("gms_points_render_frame", "opacity_raw", _set(opacity_raw=None), MESH_MODEL),
    ("gms_points_render_frame", "P_neg", _set(P=-1), "P < 0"),
    ("gms_points_render_frame", "triangles_and_P", _both(_set(triangles=None), _set(P=-1)), MESH_MODEL),
    ("gms_points_render_frame", "P_and_workspace", _both(_set(P=-1), _set(workspace_bytes=0)), "P < 0"),
    ("gms_points_render_frame", "workspace_short", _set(), WS),

    ("gms_bound_points_render_frame", "no_alloc", "alloc", NULL),
    ("gms_bound_points_render_frame", "face", _set(face=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "coeffs", _set(coeffs=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "vertices", _set(vertices=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "faces", _set(faces=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "features", _set(features=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "opacity_raw", _set(opacity_raw=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "viewmatrix", _set_settings(viewmatrix=None), MESH_MODEL),
    ("gms_bound_points_render_frame", "P_neg", _set(P=-1), BOUND_SIZES),
    ("gms_bound_points_render_frame", "F0", _set(F=0), BOUND_SIZES),
    ("gms_bound_points_render_frame", "V0", _set(V=0), BOUND_SIZES),
    ("gms_bound_points_render_frame", "face_and_F", _both(_set(face=None), _set(F=0)), MESH_MODEL),
    ("gms_bound_points_render_frame", "workspace_short", _set(), WS),

    ("gms_free_render_frame", "no_alloc", "alloc", NULL),
    ("gms_free_render_frame", "P_neg", _set(P=-1), FREE_MODEL),
    ("gms_free_render_frame", "M0", _set(M=0), FREE_MODEL),
    ("gms_free_render_frame", "M17", _set(M=17), FREE_MODEL),
    ("gms_free_render_frame", "scale_cols", _set(scale_cols=4), FREE_MODEL),
    ("gms_free_render_frame", "xyz", _set(xyz=None), FREE_MODEL),
    ("gms_free_render_frame", "rotation_raw", _set(rotation_raw=None), FREE_MODEL),
    ("gms_free_render_frame", "P0_no_tensors", _set(P=0, xyz=None, features=None), WS),
    ("gms_free_render_frame", "misaligned", _set(rotation_raw=BASE + 4), "rotation_raw must be 16-byte aligned"),
    ("gms_free_render_frame", "model_and_misaligned", _set(M=0, rotation_raw=BASE + 4), FREE_MODEL),
    ("gms_free_render_frame", "misaligned_and_workspace", _set(rotation_raw=BASE + 8, workspace_bytes=0),
     "rotation_raw must be 16-byte aligned"),
    ("gms_free_render_frame", "workspace_short", _set(), WS),

    ("gms_flame_render_frame", "no_alloc", "alloc", NULL),
    ("gms_flame_render_frame", "vertices", _set(vertices=None), MESH_MODEL),
    ("gms_flame_render_frame", "alpha", _set(alpha=None), MESH_MODEL),
    ("gms_flame_render_frame", "scaling_log", _set(scaling_log=None), MESH_MODEL),
    ("gms_flame_render_frame", "rotation_raw", _set(rotation_raw=None), MESH_MODEL),
    ("gms_flame_render_frame", "F_neg", _set(F=-1), FLAME_SIZES),
    ("gms_flame_render_frame", "K0", _set(K=0), FLAME_SIZES),
    ("gms_flame_render_frame", "V0", _set(V=0), FLAME_SIZES),
    ("gms_flame_render_frame", "M0", _set(M=0), FLAME_SIZES),
    ("gms_flame_render_frame", "M17", _set(M=17), FLAME_SIZES),
    ("gms_flame_render_frame", "FK_overflow", _set(F=1 << 16, K=1 << 15), FLAME_SIZES),
    ("gms_flame_render_frame", "misaligned", _set(rotation_raw=BASE + 12), "rotation_raw must be 16-byte aligned"),
    ("gms_flame_render_frame", "sizes_and_misaligned", _set(K=0, rotation_raw=BASE + 12), FLAME_SIZES),
    ("gms_flame_render_frame", "model_and_sizes", _set(alpha=None, M=0), MESH_MODEL),
    ("gms_flame_render_frame", "workspace_short", _set(), WS),

    ("gms_train_frame", "args", "args", NULL),
    ("gms_train_frame", "loss", _set(loss=None), NULL),
    ("gms_train_frame", "gt", _set(gt=None), NULL),
    ("gms_train_frame", "d_vertices", _set(d_vertices=None), MESH_GRADS),
    ("gms_train_frame", "d_alpha_raw", _set(d_alpha_raw=None), MESH_GRADS),
    ("gms_train_frame", "d_scale_raw", _set(d_scale_raw=None), MESH_GRADS),
    ("gms_train_frame", "d_opacity_raw", _set(d_opacity_raw=None), MESH_GRADS),
    ("gms_train_frame", "no_sh_gradient", _set(d_features=None), MESH_GRADS),
    ("gms_train_frame", "d_color_sh_only", _set(d_features=None, d_color_sh=BASE), WS),
    ("gms_train_frame", "sh_adam_only", lambda a: (_set(d_features=None)(a), _sh_adam(a)), WS),
    ("gms_train_frame", "sh_adam_m", lambda a: _sh_adam(a, m=None), "bad sh_adam"),
    ("gms_train_frame", "sh_adam_v", lambda a: _sh_adam(a, v=None), "bad sh_adam"),
    ("gms_train_frame", "sh_adam_step", lambda a: _sh_adam(a, step=0), "bad sh_adam"),
    ("gms_train_frame", "sh_adam_degree", lambda a: (_sh_adam(a), _set_settings(sh_degree=4)(a)), "bad sh_adam"),
    ("gms_train_frame", "sh_adam_degree_neg", lambda a: (_sh_adam(a), _set_settings(sh_degree=-1)(a)), "bad sh_adam"),
    ("gms_train_frame", "W0", lambda a: (_set_settings(image_width=0)(a), _set(workspace_bytes=0)(a)), WS),
    ("gms_train_frame", "model_and_grads", _set(opacity_raw=None, d_opacity_raw=None), MESH_MODEL),
    ("gms_train_frame", "grads_and_sh_adam", lambda a: (_set(d_scale_raw=None)(a), _sh_adam(a, step=0)), MESH_GRADS),
    ("gms_train_frame", "sh_adam_and_alpha", lambda a: (_sh_adam(a, v=None), _set(alpha_activation=3)(a)), "bad sh_adam"),
    ("gms_train_frame", "sh_adam_and_segments", lambda a: (_sh_adam(a, m=None), _set(n_segments=-1)(a)), "bad sh_adam"),

    ("gms_free_train_frame", "args", "args", NULL),
    ("gms_free_train_frame", "no_alloc", "alloc", NULL),
    ("gms_free_train_frame", "workspace", _set(workspace=None), NULL),
    ("gms_free_train_frame", "loss", _set(loss=None), NULL),
    ("gms_free_train_frame", "gt", _set(gt=None), NULL),
    ("gms_free_train_frame", "P_neg", _set(P=-1), FREE_MODEL),
    ("gms_free_train_frame", "M0", _set(M=0), FREE_MODEL),
    ("gms_free_train_frame", "M17", _set(M=17), FREE_MODEL),
    ("gms_free_train_frame", "scale_cols", _set(scale_cols=1), FREE_MODEL),
    ("gms_free_train_frame", "features", _set(features=None), FREE_MODEL),
    ("gms_free_train_frame", "opacity_raw", _set(opacity_raw=None), FREE_MODEL),
    ("gms_free_train_frame", "d_xyz", _set(d_xyz=None), MESH_GRADS),
    ("gms_free_train_frame", "d_scaling_raw", _set(d_scaling_raw=None), MESH_GRADS),
    ("gms_free_train_frame", "d_rotation_raw", _set(d_rotation_raw=None), MESH_GRADS),
    ("gms_free_train_frame", "d_features", _set(d_features=None), MESH_GRADS),
    ("gms_free_train_frame", "d_opacity_raw", _set(d_opacity_raw=None), MESH_GRADS),
    ("gms_free_train_frame", "P0_no_grads", _set(P=0, d_xyz=None, d_features=None, d_opacity_raw=None), WS),
    ("gms_free_train_frame", "sh_adam_only", lambda a: (_set(d_features=None)(a), _sh_adam(a)), WS),
    ("gms_free_train_frame", "accum_only", _set(accum=BASE), "accum and denom go together"),
    ("gms_free_train_frame", "denom_only", _set(denom=BASE), "accum and denom go together"),
    ("gms_free_train_frame", "accum_and_denom", _set(accum=BASE, denom=BASE), WS),
    ("gms_free_train_frame", "misaligned", _set(rotation_raw=BASE + 4),
     "rotation_raw and d_rotation_raw must be 16-byte aligned"),
    ("gms_free_train_frame", "misaligned_grad", _set(d_rotation_raw=BASE + 8),
     "rotation_raw and d_rotation_raw must be 16-byte aligned"),
    ("gms_free_train_frame", "sh_adam_m", lambda a: _sh_adam(a, m=None), "bad sh_adam"),
    ("gms_free_train_frame", "sh_adam_step", lambda a: _sh_adam(a, step=0), "bad sh_adam"),
    ("gms_free_train_frame", "sh_adam_M", lambda a: (_sh_adam(a), _set(M=9)(a)), "bad sh_adam"),
    ("gms_free_train_frame", "sh_adam_degree", lambda a: (_sh_adam(a), _set_settings(sh_degree=4)(a)), "bad sh_adam"),
    ("gms_free_train_frame", "W0", _set_settings(image_width=0), "bad image size"),
    ("gms_free_train_frame", "H_neg", _set_settings(image_height=-2), "bad image size"),
    ("gms_free_train_frame", "workspace_short", _set(), WS),
    ("gms_free_train_frame", "model_and_grads", _set(xyz=None, d_xyz=None), FREE_MODEL),
    ("gms_free_train_frame", "grads_and_accum", _set(d_opacity_raw=None, accum=BASE), MESH_GRADS),
    ("gms_free_train_frame", "accum_and_misaligned", _set(denom=BASE, rotation_raw=BASE + 4), "accum and denom go together"),
    ("gms_free_train_frame", "misaligned_and_sh_adam", lambda a: (_set(d_rotation_raw=BASE + 4)(a), _sh_adam(a, step=0)),
     "rotation_raw and d_rotation_raw must be 16-byte aligned"),
    ("gms_free_train_frame", "sh_adam_and_W", lambda a: (_sh_adam(a, v=None), _set_settings(image_width=0)(a)), "bad sh_adam"),
    ("gms_free_train_frame", "W_and_workspace", lambda a: (_set_settings(image_width=0)(a), _set(workspace_bytes=0)(a)),
     "bad image size"),
]

# The active SH degree is checked against the model's M with the model, ahead of the workspace check: a frame whose
# degree needs more coefficients than its rows hold never reaches its expansion or activation launches.
SH_RANGE = "sh_degree must be 0..3"
SH_M = "sh_degree needs more coefficients than M"
_MODEL_NULL = {"gms_render_frame": "vertices", "gms_points_render_frame": "triangles", "gms_bound_points_render_frame": "face",
               "gms_free_render_frame": "xyz", "gms_flame_render_frame": "alpha", "gms_train_frame": "vertices",
               "gms_free_train_frame": "xyz"}
_MODEL_MSG = {"gms_free_render_frame": FREE_MODEL, "gms_free_train_frame": FREE_MODEL}
for _entry in ENTRIES:
    CASES += [
        (_entry, "sh_degree_neg", _set_settings(sh_degree=-1), SH_RANGE),
        (_entry, "sh_degree_4", _set_settings(sh_degree=4), SH_RANGE),
        (_entry, "sh_degree_2_M4", lambda a: (_set(M=4)(a), _set_settings(sh_degree=2)(a)), SH_M),
        (_entry, "sh_degree_3_M15", lambda a: (_set(M=15)(a), _set_settings(sh_degree=3)(a)), SH_M),
        (_entry, "sh_degree_1_M1", lambda a: (_set(M=1)(a), _set_settings(sh_degree=1)(a)), SH_M),
        (_entry, "sh_degree_0_M1", lambda a: (_set(M=1)(a), _set_settings(sh_degree=0)(a)), WS),
        (_entry, "sh_degree_1_M4", lambda a: (_set(M=4)(a), _set_settings(sh_degree=1)(a)), WS),
        (_entry, "sh_degree_2_M9", lambda a: (_set(M=9)(a), _set_settings(sh_degree=2)(a)), WS),
        # two faults: the model check runs first, the SH degree check before the workspace check
        (_entry, "model_and_sh_degree", lambda a, t=_MODEL_NULL[_entry]: (_set(**{t: None})(a), _set_settings(sh_degree=4)(a)),
         _MODEL_MSG.get(_entry, MESH_MODEL)),
        (_entry, "sh_degree_and_workspace", lambda a: (_set(M=4, workspace_bytes=0)(a), _set_settings(sh_degree=3)(a)), SH_M),
    ]
CASES += [
    # with sh_adam the SH Adam check owns the degree range, as before
    ("gms_train_frame", "sh_adam_and_sh_degree_M", lambda a: (_sh_adam(a, step=0), _set(M=4)(a)), "bad sh_adam"),
    ("gms_free_train_frame", "sh_degree_M_and_W", lambda a: (_set(M=4)(a), _set_settings(image_width=0)(a)), SH_M),
]


def _noop_alloc():
    return _lib.ALLOC_FN(lambda user, which, n: 0)


@pytest.mark.parametrize("entry,case,mutate,message", CASES, ids=[f"{c[0]}-{c[1]}" for c in CASES])
def test_refusal(entry, case, mutate, message):
    L = _lib.lib()
    a = ENTRIES[entry]()
    cb = _noop_alloc()
    if mutate == "alloc":
        cb = _lib.ALLOC_FN()        # NULL
    keep = None if isinstance(mutate, str) else mutate(a)       # host arrays the struct points at stay alive
    rc = getattr(L, entry)(None if mutate == "args" else C.byref(a), cb, None, None)
    del keep
    assert rc == _lib.GMS_E_ARG
    assert L.gms_last_error().decode() == f"{entry}: {message}"


GRID = [(0, 16, 16), (1, 1, 1), (7, 33, 17), (1000, 64, 48), (123457, 1920, 1080)]
FRAME_BYTES = [19968, 4608, 39936, 302336, 145553408]
RENDER_BYTES = [1536, 1536, 1536, 44800, 5433600]
# gms_frame_views offsets from a workspace at BASE + 40: xyz, scales, rotations, opacities, radii, image, invdepth
VIEW_OFFSETS = [(256, 512, 768, 1024, 1280, 1536, 4608), (256, 512, 768, 1024, 1280, 1536, 1792),
                (256, 512, 768, 1024, 1280, 1536, 8448), (256, 12288, 24320, 40448, 44544, 48640, 85504),
                (256, 1481984, 2963712, 4939264, 5433344, 5927424, 30810624)]


@pytest.mark.parametrize("i", range(len(GRID)))
def test_workspace_sizes(i):
    L = _lib.lib()
    P, W, H = GRID[i]
    assert L.gms_frame_workspace_bytes(P, W, H) == FRAME_BYTES[i]
    for fn in ("gms_render_workspace_bytes", "gms_points_render_workspace_bytes", "gms_bound_points_render_workspace_bytes",
               "gms_flame_render_workspace_bytes"):
        assert getattr(L, fn)(P, W, H) == RENDER_BYTES[i], fn
    v = _lib.FrameView()
    assert L.gms_frame_views(BASE + 40, P, W, H, C.byref(v)) == _lib.GMS_OK
    assert tuple(getattr(v, n) - BASE for n, _ in _lib.FrameView._fields_) == VIEW_OFFSETS[i]
