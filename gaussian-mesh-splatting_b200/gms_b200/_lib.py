"""ctypes binding of libgms_b200.so (C ABI declared in include/gms_b200.h).

The product path REQUIRES the CUDA library: there is no CPU or PyTorch fallback.  Importing this module
is cheap; the first call that needs the library raises GmsLibraryError if it has not been built
(`python -c "import __graft_entry__ as g; g.build()"` or `python gaussian-mesh-splatting_b200/build.py`).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgms_b200.so")

ALPHA_RELU, ALPHA_SOFTMAX = 0, 1   # gms_*_args.alpha_activation: relu + 1e-8, normalised (gs_mesh); softmax (gs_flame)
FORWARD_ONLY = 1        # gms_raster_outputs.flags: no backward will follow (skip the survivor lists)
GMS_OK, GMS_E_ARG, GMS_E_CUDA, GMS_E_ALLOC, GMS_E_UNSUPPORTED, GMS_E_DEBUG = 0, -1, -2, -3, -4, -5
BUF_GEOM, BUF_BINNING, BUF_IMAGE = 0, 1, 2

c_float_p = C.c_void_p   # raw device pointers travel as integers


class GmsLibraryError(RuntimeError):
    pass


class RasterSettings(C.Structure):
    _fields_ = [("image_height", C.c_int32), ("image_width", C.c_int32), ("tanfovx", C.c_float),
                ("tanfovy", C.c_float), ("bg", C.c_void_p), ("scale_modifier", C.c_float),
                ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("sh_degree", C.c_int32),
                ("campos", C.c_void_p), ("prefiltered", C.c_int32), ("debug", C.c_int32),
                ("antialiasing", C.c_int32)]


class RasterInputs(C.Structure):
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("means3D", C.c_void_p), ("opacities", C.c_void_p),
                ("shs", C.c_void_p), ("colors_precomp", C.c_void_p), ("scales", C.c_void_p),
                ("rotations", C.c_void_p), ("cov3D_precomp", C.c_void_p)]


class RasterOutputs(C.Structure):
    _fields_ = [("out_color", C.c_void_p), ("radii", C.c_void_p), ("out_invdepth", C.c_void_p), ("flags", C.c_int32)]


class RasterSaved(C.Structure):
    _fields_ = [("geom", C.c_void_p), ("binning", C.c_void_p), ("image", C.c_void_p),
                ("num_rendered", C.c_int64), ("num_visible", C.c_int64), ("binning_capacity", C.c_int64),
                ("flags", C.c_int32)]


class RasterGrads(C.Structure):
    _fields_ = [("dL_dmeans3D", C.c_void_p), ("dL_dmeans2D", C.c_void_p), ("dL_dopacities", C.c_void_p),
                ("dL_dshs", C.c_void_p), ("dL_dcolors_precomp", C.c_void_p), ("dL_dscales", C.c_void_p),
                ("dL_drotations", C.c_void_p), ("dL_dcov3D_precomp", C.c_void_p), ("dL_dcolors_sh", C.c_void_p)]


class DebugViews(C.Structure):
    _fields_ = [("means2D", C.c_void_p), ("depths", C.c_void_p), ("cov3D", C.c_void_p),
                ("conic_opacity", C.c_void_p), ("rgb", C.c_void_p), ("clamped", C.c_void_p),
                ("tiles_touched", C.c_void_p), ("point_list", C.c_void_p), ("tile_keys", C.c_void_p),
                ("ranges", C.c_void_p), ("final_T", C.c_void_p), ("n_contrib", C.c_void_p), ("dgeom", C.c_void_p),
                ("surv", C.c_void_p), ("nsurv", C.c_void_p)]


class ExpandArgs(C.Structure):
    _fields_ = [("V", C.c_int32), ("F", C.c_int32), ("K", C.c_int32), ("vertices", C.c_void_p),
                ("faces", C.c_void_p), ("triangles_in", C.c_void_p), ("alpha_raw", C.c_void_p),
                ("scale_raw", C.c_void_p), ("eps", C.c_float), ("alpha", C.c_void_p),
                ("triangles", C.c_void_p), ("xyz", C.c_void_p), ("scaling_log", C.c_void_p),
                ("rotation_raw", C.c_void_p), ("scaling_act", C.c_void_p), ("rotation_act", C.c_void_p),
                ("alpha_activation", C.c_int32)]


class ExpandGrads(C.Structure):
    _fields_ = [("dL_dxyz", C.c_void_p), ("dL_dscaling_log", C.c_void_p), ("dL_drotation_raw", C.c_void_p),
                ("dL_dscaling_act", C.c_void_p), ("dL_drotation_act", C.c_void_p),
                ("dL_dvertices", C.c_void_p), ("dL_dtriangles", C.c_void_p), ("dL_dalpha_raw", C.c_void_p),
                ("dL_dscale_raw", C.c_void_p)]


class PointsArgs(C.Structure):
    _fields_ = [("P", C.c_int32), ("triangles", C.c_void_p), ("eps", C.c_float), ("xyz", C.c_void_p),
                ("scaling_log", C.c_void_p), ("rotation_raw", C.c_void_p), ("scaling_act", C.c_void_p),
                ("rotation_act", C.c_void_p)]


class PointsVerticesArgs(C.Structure):
    """struct gms_points_vertices_args"""
    _fields_ = [("P", C.c_int32), ("xyz", C.c_void_p), ("scaling_log", C.c_void_p), ("scaling_cols", C.c_int32),
                ("rotation_raw", C.c_void_p), ("triangles", C.c_void_p)]


class LossArgs(C.Structure):
    _fields_ = [("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("img", C.c_void_p), ("gt", C.c_void_p),
                ("lambda_dssim", C.c_float), ("dL_dloss", C.c_void_p), ("loss", C.c_void_p), ("dL_dimg", C.c_void_p),
                ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


class AdamArgs(C.Structure):
    _fields_ = [("n", C.c_int64), ("offset", C.c_int64), ("p", C.c_void_p), ("g", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p),
                ("nseg", C.c_int32), ("seg_end", C.c_int64 * 8), ("lr0", C.c_double * 8), ("lr1", C.c_double * 8),
                ("inner", C.c_int32 * 8), ("period", C.c_int32 * 8), ("beta1", C.c_double), ("beta2", C.c_double),
                ("eps", C.c_double), ("step", C.c_int32), ("zero_grad", C.c_int32), ("zero_end", C.c_int64)]


class ShAdam(C.Structure):
    """struct gms_sh_adam"""
    _fields_ = [("m", C.c_void_p), ("v", C.c_void_p), ("lr_dc", C.c_double), ("lr_rest", C.c_double), ("beta1", C.c_double),
                ("beta2", C.c_double), ("eps", C.c_double), ("step", C.c_int32)]


class MeshSegment(C.Structure):
    """struct gms_mesh_segment"""
    _fields_ = [("F", C.c_int32), ("K", C.c_int32)]


def mesh_segments(segments) -> "C.Array":
    """[(F_i, K_i), ...] -> the host array gms_frame_args / gms_render_args point `segments` at."""
    arr = (MeshSegment * len(segments))()
    for i, (F, K) in enumerate(segments):
        arr[i].F, arr[i].K = int(F), int(K)
    return arr


class FrameArgs(C.Structure):
    _fields_ = [("V", C.c_int32), ("F", C.c_int32), ("K", C.c_int32), ("M", C.c_int32),
                ("vertices", C.c_void_p), ("faces", C.c_void_p), ("alpha_raw", C.c_void_p), ("scale_raw", C.c_void_p),
                ("features", C.c_void_p), ("opacity_raw", C.c_void_p), ("eps", C.c_float),
                ("d_vertices", C.c_void_p), ("d_alpha_raw", C.c_void_p), ("d_scale_raw", C.c_void_p),
                ("d_features", C.c_void_p), ("d_opacity_raw", C.c_void_p),
                ("settings", RasterSettings), ("gt", C.c_void_p), ("lambda_dssim", C.c_float), ("loss", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("num_rendered", C.POINTER(C.c_int64)),
                ("binning_capacity", C.c_int64), ("n_host_mapped", C.c_void_p), ("d_color_sh", C.c_void_p),
                ("event_sh_ready", C.c_void_p), ("event_loss_ready", C.c_void_p), ("sh_adam", C.POINTER(ShAdam)),
                ("segments", C.POINTER(MeshSegment)), ("n_segments", C.c_int32), ("anomaly_stages", C.c_uint32),
                ("anomaly", C.c_void_p), ("alpha_activation", C.c_int32)]


class FrameView(C.Structure):
    _fields_ = [("xyz", C.c_void_p), ("scales", C.c_void_p), ("rotations", C.c_void_p), ("opacities", C.c_void_p),
                ("radii", C.c_void_p), ("image", C.c_void_p), ("invdepth", C.c_void_p)]


class RenderArgs(C.Structure):
    """struct gms_render_args"""
    _fields_ = [("V", C.c_int32), ("F", C.c_int32), ("K", C.c_int32), ("M", C.c_int32),
                ("vertices", C.c_void_p), ("faces", C.c_void_p), ("alpha_raw", C.c_void_p), ("scale_raw", C.c_void_p),
                ("features", C.c_void_p), ("opacity_raw", C.c_void_p), ("eps", C.c_float), ("settings", RasterSettings),
                ("image", C.c_void_p), ("invdepth", C.c_void_p), ("radii", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("num_rendered", C.POINTER(C.c_int64)),
                ("binning_capacity", C.c_int64), ("n_host_mapped", C.c_void_p),
                ("segments", C.POINTER(MeshSegment)), ("n_segments", C.c_int32), ("alpha_activation", C.c_int32)]


class FlameRenderArgs(C.Structure):
    """struct gms_flame_render_args"""
    _fields_ = [("V", C.c_int32), ("F", C.c_int32), ("K", C.c_int32), ("M", C.c_int32), ("vertices", C.c_void_p), ("faces", C.c_void_p),
                ("alpha", C.c_void_p), ("scaling_log", C.c_void_p), ("rotation_raw", C.c_void_p), ("features", C.c_void_p),
                ("opacity_raw", C.c_void_p), ("settings", RasterSettings), ("image", C.c_void_p), ("invdepth", C.c_void_p),
                ("radii", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
                ("num_rendered", C.POINTER(C.c_int64)), ("binning_capacity", C.c_int64), ("n_host_mapped", C.c_void_p)]


class PointsRenderArgs(C.Structure):
    """struct gms_points_render_args"""
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("triangles", C.c_void_p), ("features", C.c_void_p),
                ("opacity_raw", C.c_void_p), ("eps", C.c_float), ("settings", RasterSettings),
                ("image", C.c_void_p), ("invdepth", C.c_void_p), ("radii", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("num_rendered", C.POINTER(C.c_int64)),
                ("binning_capacity", C.c_int64), ("n_host_mapped", C.c_void_p)]


class PseudomeshBindArgs(C.Structure):
    """struct gms_pseudomesh_bind_args"""
    _fields_ = [("P", C.c_int32), ("triangles", C.c_void_p), ("V", C.c_int32), ("F", C.c_int32), ("vertices", C.c_void_p),
                ("faces", C.c_void_p), ("face", C.c_void_p), ("coeffs", C.c_void_p), ("n_degenerate", C.POINTER(C.c_int32)),
                ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


class PseudomeshReposeArgs(C.Structure):
    """struct gms_pseudomesh_repose_args"""
    _fields_ = [("P", C.c_int32), ("face", C.c_void_p), ("coeffs", C.c_void_p), ("V", C.c_int32), ("F", C.c_int32),
                ("vertices", C.c_void_p), ("faces", C.c_void_p), ("triangles", C.c_void_p)]


class BoundPointsRenderArgs(C.Structure):
    """struct gms_bound_points_render_args"""
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("face", C.c_void_p), ("coeffs", C.c_void_p), ("V", C.c_int32),
                ("F", C.c_int32), ("vertices", C.c_void_p), ("faces", C.c_void_p), ("features", C.c_void_p),
                ("opacity_raw", C.c_void_p), ("eps", C.c_float), ("settings", RasterSettings),
                ("image", C.c_void_p), ("invdepth", C.c_void_p), ("radii", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("num_rendered", C.POINTER(C.c_int64)),
                ("binning_capacity", C.c_int64), ("n_host_mapped", C.c_void_p)]


class FreeFrameArgs(C.Structure):
    """struct gms_free_frame_args"""
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("scale_cols", C.c_int32), ("xyz", C.c_void_p), ("scaling_raw", C.c_void_p),
                ("rotation_raw", C.c_void_p), ("features", C.c_void_p), ("opacity_raw", C.c_void_p), ("eps", C.c_float),
                ("d_xyz", C.c_void_p), ("d_scaling_raw", C.c_void_p), ("d_rotation_raw", C.c_void_p), ("d_features", C.c_void_p),
                ("d_opacity_raw", C.c_void_p), ("accum", C.c_void_p), ("denom", C.c_void_p), ("settings", RasterSettings),
                ("gt", C.c_void_p), ("lambda_dssim", C.c_float), ("loss", C.c_void_p), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t), ("num_rendered", C.POINTER(C.c_int64)), ("binning_capacity", C.c_int64),
                ("n_host_mapped", C.c_void_p), ("event_loss_ready", C.c_void_p), ("sh_adam", C.POINTER(ShAdam)),
                ("anomaly", C.c_void_p), ("anomaly_stages", C.c_uint32)]


class FreeRenderArgs(C.Structure):
    """struct gms_free_render_args"""
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("scale_cols", C.c_int32), ("xyz", C.c_void_p), ("scaling_raw", C.c_void_p),
                ("rotation_raw", C.c_void_p), ("features", C.c_void_p), ("opacity_raw", C.c_void_p), ("eps", C.c_float),
                ("settings", RasterSettings), ("image", C.c_void_p), ("invdepth", C.c_void_p), ("radii", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("num_rendered", C.POINTER(C.c_int64)),
                ("binning_capacity", C.c_int64), ("n_host_mapped", C.c_void_p)]


FATE_CLONE, FATE_SPLIT, FATE_PRUNE, FATE_PRUNE_CHILDREN = 1, 2, 4, 8     # gms_densify_plan_args.fate bits


class DensifyPlanArgs(C.Structure):
    """struct gms_densify_plan_args"""
    _fields_ = [("P", C.c_int32), ("scale_cols", C.c_int32), ("accum", C.c_void_p), ("denom", C.c_void_p),
                ("scaling_raw", C.c_void_p), ("opacity_raw", C.c_void_p), ("eps", C.c_float), ("grad_threshold", C.c_float),
                ("split_scale", C.c_float), ("min_opacity", C.c_float), ("max_world_scale", C.c_float), ("fate", C.c_void_p),
                ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t), ("result", C.POINTER(C.c_int32))]


class FreeSet(C.Structure):
    """struct gms_free_set"""
    _fields_ = [("xyz", C.c_void_p), ("scaling", C.c_void_p), ("rotation", C.c_void_p), ("opacity", C.c_void_p),
                ("features", C.c_void_p)]


class DensifyApplyArgs(C.Structure):
    """struct gms_densify_apply_args"""
    _fields_ = [("P", C.c_int32), ("new_P", C.c_int32), ("scale_cols", C.c_int32), ("M", C.c_int32), ("eps", C.c_float),
                ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t), ("result", C.POINTER(C.c_int32)),
                ("normals", C.c_void_p), ("src", FreeSet * 3), ("dst", FreeSet * 3)]


class MetricsArgs(C.Structure):
    """struct gms_metrics_args"""
    _fields_ = [("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("img", C.c_void_p), ("gt", C.c_void_p),
                ("quantize", C.c_int32), ("out", C.c_void_p), ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


LPIPS_WEIGHT_FLOATS = 14716480    # GMS_LPIPS_WEIGHT_FLOATS


class LpipsArgs(C.Structure):
    """struct gms_lpips_args"""
    _fields_ = [("H", C.c_int32), ("W", C.c_int32), ("img", C.c_void_p), ("gt", C.c_void_p), ("weights", C.c_void_p),
                ("out", C.c_void_p), ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


class AdamShArgs(C.Structure):
    _fields_ = [("P", C.c_int32), ("M", C.c_int32), ("sh_degree", C.c_int32), ("R", C.c_int32), ("xyz", C.c_void_p),
                ("exchange", C.c_void_p), ("slot_floats", C.c_int64), ("grad_scale", C.c_float), ("p", C.c_void_p),
                ("m", C.c_void_p), ("v", C.c_void_p), ("lr_dc", C.c_double), ("lr_rest", C.c_double), ("beta1", C.c_double),
                ("beta2", C.c_double), ("eps", C.c_double), ("step", C.c_int32)]


class ResizeArgs(C.Structure):
    """struct gms_resize_args"""
    _fields_ = [("in_w", C.c_int32), ("in_h", C.c_int32), ("out_w", C.c_int32), ("out_h", C.c_int32), ("C", C.c_int32),
                ("src", C.c_void_p), ("dst", C.c_void_p), ("bounds_h", C.c_void_p), ("coeffs_h", C.c_void_p), ("ksize_h", C.c_int32),
                ("bounds_v", C.c_void_p), ("coeffs_v", C.c_void_p), ("ksize_v", C.c_int32), ("row0", C.c_int32), ("rows", C.c_int32),
                ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


KNN_BOX = 64        # GMS_KNN_BOX: points per box of the three-nearest-neighbour search


class KnnArgs(C.Structure):
    """struct gms_knn_args"""
    _fields_ = [("P", C.c_int32), ("points", C.c_void_p), ("dist2", C.c_void_p), ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


ALPHA_BUF_SCRATCH, ALPHA_BUF_LISTS, ALPHA_BUF_FACES, ALPHA_BUF_INDEX = 0, 1, 2, 3     # GMS_ALPHA_BUF_*: gms_alpha_shape's allocations
ALPHA_LIST_CAP = 256        # GMS_ALPHA_LIST_CAP: 3-alpha list entries staged in shared memory per point
NORMALS_MAX_NN = 64         # GMS_NORMALS_MAX_NN


class AlphaShapeArgs(C.Structure):
    """struct gms_alpha_shape_args"""
    _fields_ = [("P", C.c_int32), ("points", C.c_void_p), ("alpha", C.c_double), ("n_faces", C.POINTER(C.c_int64)),
                ("n_vertices", C.POINTER(C.c_int64))]


class NormalsArgs(C.Structure):
    """struct gms_normals_args"""
    _fields_ = [("P", C.c_int32), ("points", C.c_void_p), ("radius", C.c_double), ("max_nn", C.c_int32), ("normals", C.c_void_p),
                ("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t)]


FLAME_JOINTS = 5    # GMS_FLAME_JOINTS


class FlameLbsArgs(C.Structure):
    """struct gms_flame_lbs_args"""
    _fields_ = [("V", C.c_int32), ("n_shape", C.c_int32), ("n_exp", C.c_int32), ("n_joints", C.c_int32),
                ("parents", C.c_int32 * FLAME_JOINTS)] + \
               [(n, C.c_void_p) for n in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights", "shape", "expression",
                                          "pose", "neck_pose", "transl", "enlargement", "vertices", "vertices_grad", "d_shape",
                                          "d_expression", "d_pose", "d_neck_pose", "d_transl", "d_enlargement", "workspace")] + \
               [("workspace_bytes", C.c_size_t)]


ANOMALY_NONE = (1 << 64) - 1        # GMS_ANOMALY_NONE: the record of a scan that found no NaN
# GMS_ANOMALY_*: the stages, in the order a frame runs them, and the tensors of each
(ANOMALY_LOSS, ANOMALY_COMPOSITE_BWD, ANOMALY_PREPROCESS_BWD, ANOMALY_EXPAND_BWD, ANOMALY_ACTIVATION_BWD,
 ANOMALY_FLAME_BWD) = range(6)
ANOMALY_STAGES = 6
ANOMALY_DIMAGE = 0
ANOMALY_DGEOM = 0
(ANOMALY_DMEANS3D, ANOMALY_DSCALES, ANOMALY_DROTATIONS, ANOMALY_DOPACITY_RAW, ANOMALY_DSHS, ANOMALY_DCOLOR_SH) = range(6)
ANOMALY_DVERTICES, ANOMALY_DALPHA_RAW, ANOMALY_DSCALE_RAW = range(3)
ANOMALY_DSCALING_RAW, ANOMALY_DROTATION_RAW, ANOMALY_ACCUM = range(3)
(ANOMALY_DSHAPE, ANOMALY_DEXPRESSION, ANOMALY_DPOSE, ANOMALY_DNECK_POSE, ANOMALY_DTRANSL, ANOMALY_DENLARGEMENT) = range(6)
NAN_SCAN_MAX_BUFFERS = 8            # GMS_NAN_SCAN_MAX_BUFFERS


class NanBuffer(C.Structure):
    """struct gms_nan_buffer"""
    _fields_ = [("ptr", C.c_void_p), ("n", C.c_int64), ("tensor", C.c_int32)]


class NanScanArgs(C.Structure):
    """struct gms_nan_scan_args"""
    _fields_ = [("buffers", NanBuffer * NAN_SCAN_MAX_BUFFERS), ("n_buffers", C.c_int32), ("stage", C.c_int32),
                ("record", C.c_void_p)]


DEBUG_NONE = (1 << 64) - 1        # GMS_DEBUG_NONE: the key of a binning check that found no violation
DEBUG_ORDER, DEBUG_RANGES, DEBUG_GAUSSIAN, DEBUG_SURVIVOR = 1, 2, 3, 4     # GMS_DEBUG_*: the checks (key >> 56)


class DebugBinsArgs(C.Structure):
    """struct gms_debug_bins_args"""
    _fields_ = [("P", C.c_int32), ("tiles_x", C.c_int32), ("tiles_y", C.c_int32), ("n", C.c_int64), ("point_list", C.c_void_p),
                ("tile_keys", C.c_void_p), ("key_bits", C.c_int32), ("ranges", C.c_void_p), ("radii", C.c_void_p),
                ("rect", C.c_void_p), ("depth_keys", C.c_void_p), ("surv", C.c_void_p), ("nsurv", C.c_void_p),
                ("key", C.POINTER(C.c_uint64))]


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_int, C.c_size_t)

# every symbol include/gms_b200.h declares (tests/test_abi.py checks the library exports all of them)
ABI_SYMBOLS = ["gms_scratch_bytes", "gms_binning_bytes", "gms_rasterize_forward", "gms_rasterize_forward_nosync", "gms_rasterize_backward",
               "gms_mark_visible", "gms_debug_get_views", "gms_debug_unpack", "gms_expand_forward",
               "gms_expand_backward", "gms_last_error", "gms_version", "gms_launch_count", "gms_set_option",
               "gms_kernel_times", "gms_loss_scratch_bytes", "gms_l1_ssim_loss", "gms_adam_step",
               "gms_frame_workspace_bytes", "gms_train_frame", "gms_points_expand_forward",
               "gms_points_prepare_vertices", "gms_image_quantize", "gms_image_clamp_u8", "gms_image_dequantize", "gms_adam_sh_factored", "gms_frame_views",
               "gms_render_workspace_bytes", "gms_render_frame", "gms_metrics_scratch_bytes", "gms_image_metrics",
               "gms_points_render_workspace_bytes", "gms_points_render_frame", "gms_pseudomesh_bind_scratch_bytes",
               "gms_pseudomesh_bind", "gms_pseudomesh_repose", "gms_bound_points_render_workspace_bytes",
               "gms_bound_points_render_frame", "gms_free_train_frame", "gms_free_render_frame", "gms_densify_scratch_bytes",
               "gms_densify_plan", "gms_densify_apply", "gms_knn_scratch_bytes", "gms_knn_dist2",
               "gms_flame_render_workspace_bytes", "gms_flame_render_frame", "gms_image_composite_rgba", "gms_image_resize_u8",
               "gms_flame_lbs_workspace_bytes", "gms_flame_lbs_forward", "gms_flame_lbs_backward", "gms_lpips_scratch_bytes",
               "gms_lpips_vgg", "gms_alpha_shape", "gms_normals_scratch_bytes", "gms_estimate_normals", "gms_nan_scan",
               "gms_debug_check_bins"]

_lib = None


def lib():
    """Load libgms_b200.so; fail loudly if it is missing (no fallback path exists by design)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GmsLibraryError(
            f"{LIB_PATH} not found: the CUDA extension has not been built. Run "
            f"`python gaussian-mesh-splatting_b200/build.py` (needs nvcc, sm_90a). There is no CPU fallback.")
    try:
        L = C.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise GmsLibraryError(f"cannot load {LIB_PATH}: {e}") from e
    L.gms_last_error.restype = C.c_char_p
    L.gms_version.restype = C.c_char_p
    L.gms_launch_count.restype = C.c_int64
    L.gms_launch_count.argtypes = [C.c_int]
    L.gms_binning_bytes.restype = C.c_size_t
    L.gms_binning_bytes.argtypes = [C.c_int64, C.c_int32]
    L.gms_scratch_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.gms_rasterize_forward.argtypes = [C.POINTER(RasterSettings), C.POINTER(RasterInputs), C.POINTER(RasterOutputs),
                                        ALLOC_FN, C.c_void_p, C.POINTER(RasterSaved), C.c_void_p]
    L.gms_rasterize_forward_nosync.argtypes = [C.POINTER(RasterSettings), C.POINTER(RasterInputs), C.POINTER(RasterOutputs),
                                               ALLOC_FN, C.c_void_p, C.POINTER(RasterSaved), C.c_int64, C.c_void_p, C.c_void_p]
    L.gms_rasterize_backward.argtypes = [C.POINTER(RasterSettings), C.POINTER(RasterInputs), C.c_void_p,
                                         C.POINTER(RasterSaved), C.c_void_p, C.c_void_p, C.POINTER(RasterGrads),
                                         C.c_void_p]
    L.gms_mark_visible.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gms_debug_get_views.argtypes = [C.POINTER(RasterSaved), C.c_int32, C.c_int32, C.c_int32, C.POINTER(DebugViews)]
    L.gms_debug_unpack.argtypes = [C.POINTER(RasterSaved), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    L.gms_expand_forward.argtypes = [C.POINTER(ExpandArgs), C.c_void_p]
    L.gms_expand_backward.argtypes = [C.POINTER(ExpandArgs), C.POINTER(ExpandGrads), C.c_void_p]
    L.gms_set_option.argtypes = [C.c_char_p, C.c_int]
    L.gms_loss_scratch_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]
    L.gms_l1_ssim_loss.argtypes = [C.POINTER(LossArgs), C.c_void_p]
    L.gms_adam_step.argtypes = [C.POINTER(AdamArgs), C.c_void_p]
    L.gms_points_expand_forward.argtypes = [C.POINTER(PointsArgs), C.c_void_p]
    L.gms_points_prepare_vertices.argtypes = [C.POINTER(PointsVerticesArgs), C.c_void_p]
    L.gms_image_quantize.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    L.gms_image_clamp_u8.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    L.gms_image_dequantize.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    L.gms_image_composite_rgba.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    L.gms_image_resize_u8.argtypes = [C.POINTER(ResizeArgs), C.c_void_p]
    L.gms_adam_sh_factored.argtypes = [C.POINTER(AdamShArgs), C.c_void_p]
    L.gms_frame_views.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(FrameView)]
    L.gms_frame_workspace_bytes.restype = C.c_size_t
    L.gms_frame_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.gms_train_frame.argtypes = [C.POINTER(FrameArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_render_workspace_bytes.restype = C.c_size_t
    L.gms_render_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.gms_render_frame.argtypes = [C.POINTER(RenderArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_flame_render_workspace_bytes.restype = C.c_size_t
    L.gms_flame_render_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.gms_flame_render_frame.argtypes = [C.POINTER(FlameRenderArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_points_render_workspace_bytes.restype = C.c_size_t
    L.gms_points_render_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.gms_points_render_frame.argtypes = [C.POINTER(PointsRenderArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_pseudomesh_bind_scratch_bytes.restype = C.c_size_t
    L.gms_pseudomesh_bind_scratch_bytes.argtypes = [C.c_int32]
    L.gms_pseudomesh_bind.argtypes = [C.POINTER(PseudomeshBindArgs), C.c_void_p]
    L.gms_pseudomesh_repose.argtypes = [C.POINTER(PseudomeshReposeArgs), C.c_void_p]
    L.gms_bound_points_render_workspace_bytes.restype = C.c_size_t
    L.gms_bound_points_render_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.gms_bound_points_render_frame.argtypes = [C.POINTER(BoundPointsRenderArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_free_train_frame.argtypes = [C.POINTER(FreeFrameArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_free_render_frame.argtypes = [C.POINTER(FreeRenderArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_densify_scratch_bytes.restype = C.c_size_t
    L.gms_densify_scratch_bytes.argtypes = [C.c_int32]
    L.gms_densify_plan.argtypes = [C.POINTER(DensifyPlanArgs), C.c_void_p]
    L.gms_densify_apply.argtypes = [C.POINTER(DensifyApplyArgs), C.c_void_p]
    L.gms_knn_scratch_bytes.restype = C.c_size_t
    L.gms_knn_scratch_bytes.argtypes = [C.c_int32]
    L.gms_knn_dist2.argtypes = [C.POINTER(KnnArgs), C.c_void_p]
    L.gms_flame_lbs_workspace_bytes.restype = C.c_size_t
    L.gms_flame_lbs_workspace_bytes.argtypes = [C.c_int32]
    L.gms_flame_lbs_forward.argtypes = [C.POINTER(FlameLbsArgs), C.c_void_p]
    L.gms_flame_lbs_backward.argtypes = [C.POINTER(FlameLbsArgs), C.c_void_p]
    L.gms_metrics_scratch_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]
    L.gms_image_metrics.argtypes = [C.POINTER(MetricsArgs), C.c_void_p]
    L.gms_lpips_scratch_bytes.restype = C.c_size_t
    L.gms_lpips_scratch_bytes.argtypes = [C.c_int32, C.c_int32]
    L.gms_lpips_vgg.argtypes = [C.POINTER(LpipsArgs), C.c_void_p]
    L.gms_alpha_shape.argtypes = [C.POINTER(AlphaShapeArgs), ALLOC_FN, C.c_void_p, C.c_void_p]
    L.gms_normals_scratch_bytes.restype = C.c_size_t
    L.gms_normals_scratch_bytes.argtypes = [C.c_int32]
    L.gms_estimate_normals.argtypes = [C.POINTER(NormalsArgs), C.c_void_p]
    L.gms_nan_scan.argtypes = [C.POINTER(NanScanArgs), C.c_void_p]
    L.gms_debug_check_bins.argtypes = [C.POINTER(DebugBinsArgs), C.c_void_p]
    _lib = L
    # GMS_OPTIONS="key=value,key=value": tuning knobs applied at load (A/B runs of whole test suites / benches)
    for kv in filter(None, os.environ.get("GMS_OPTIONS", "").split(",")):
        k, _, v = kv.partition("=")
        if L.gms_set_option(k.strip().encode(), int(v)) == -1:
            raise GmsLibraryError(f"GMS_OPTIONS: unknown option {k!r}")
    return L


def check(rc: int, what: str) -> None:
    if rc != GMS_OK:
        msg = lib().gms_last_error().decode("utf-8", "replace")
        if rc == GMS_E_ARG:
            # same exception type/text as the stock Python shim for bad argument combinations
            raise Exception(msg)
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


def set_option(key: str, value: int) -> int:
    return int(lib().gms_set_option(key.encode(), int(value)))


def kernel_times(reset: bool = True) -> dict:
    """{kernel name: (accumulated ms, launches)} measured by CUDA events on the launching stream."""
    L = lib()
    n = 32
    ms = (C.c_double * n)(); cnt = (C.c_int64 * n)(); names = (C.c_char_p * n)()
    k = L.gms_kernel_times(1 if reset else 0, n, ms, cnt, names)
    return {names[i].decode(): (float(ms[i]), int(cnt[i])) for i in range(min(k, n)) if names[i]}


def launch_count(reset: bool = False) -> int:
    return int(lib().gms_launch_count(1 if reset else 0))
