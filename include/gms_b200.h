/*
 * gms_b200.h -- C ABI of libgms_b200.so, the H100-native (sm_90a) mesh-Gaussian rasterizer.
 *
 * This is the drop-in boundary for the ONE hot path of waczjoan/gaussian-mesh-splatting:
 *   mesh -> Gaussian expansion, preprocess (3D->2D + SH), tile binning/sort, per-tile alpha
 *   compositing forward and backward.
 * Plain C: raw DEVICE pointers, sizes, a cudaStream_t passed as void*.  No torch types.
 * Every function returns 0 on success, a negative GMS_E_* code otherwise; gms_last_error()
 * returns a human-readable message for the calling thread's last failure.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference; the rasterizer
 * itself is the un-vendored submodule submodules/diff-gaussian-rasterization, so for it the cited lines
 * are the reference's CALL SITES and [upstream] names the function of graphdeco-inria/diff-gaussian-rasterization
 * that the reference's pybind module `diff_gaussian_rasterization._C` exports):
 *
 *   gms_rasterize_forward    <- _C.rasterize_gaussians            [upstream rasterize_points.cu: RasterizeGaussiansCUDA]
 *                               reached from renderer/gaussian_renderer/__init__.py:94-102 (and :104-112, :97-105,
 *                               :99-107 of the animated / points / flame renderers)
 *   gms_rasterize_backward   <- _C.rasterize_gaussians_backward   [upstream RasterizeGaussiansBackwardCUDA]
 *                               reached from loss.backward(), train.py:108
 *   gms_mark_visible         <- _C.mark_visible                   [upstream markVisible]
 *   gms_expand_forward       <- GaussianMeshModel.update_alpha + _calc_xyz + prepare_scaling_rot + rot_to_quat_batch
 *                               games/mesh_splatting/scene/gaussian_mesh_model.py:86-169, utils/general_utils.py:19-96,
 *                               and the activation getters scene/gaussian_model.py:95-115 (optional fused outputs)
 *   gms_expand_backward      <- the autograd graph of the above (train.py:108 -> vertices/_alpha/_scale .grad)
 *
 * Scratch memory follows the stock extension's ownership model: the CALLER owns every byte.  The library
 * asks for its three scratch regions (per-Gaussian "geom", per-duplicate "binning", per-pixel "image")
 * through a callback, exactly like the resize-lambdas the stock _C module hands to CudaRasterizer
 * [upstream rasterize_points.cu: resizeFunctional]; the Python shim serves them from torch uint8 tensors
 * and keeps them alive for backward (ctx.save_for_backward in the stock shim).
 */
/* Threading: the library keeps per-PROCESS state (tuning options, launch counter, kernel timers, the pinned word the
 * synchronising forward reads N through).  Calls must come from one host thread at a time; concurrent calls from several
 * threads -- or interleaving a forward on one stream with option changes -- are not supported (the stock extension has
 * the same restriction: it launches on the legacy default stream and blocks on a cudaMemcpy).  Use one process per GPU,
 * as bench.py / torchrun do.  Error strings (gms_last_error) are per thread. */
#ifndef GMS_B200_H
#define GMS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GMS_OK 0
#define GMS_E_ARG (-1)        /* bad argument combination (e.g. both shs and colors_precomp) */
#define GMS_E_CUDA (-2)       /* a CUDA call or launch failed; see gms_last_error() */
#define GMS_E_ALLOC (-3)      /* the allocation callback returned NULL */
#define GMS_E_UNSUPPORTED (-4)

#define GMS_BUF_GEOM 0
#define GMS_BUF_BINNING 1
#define GMS_BUF_IMAGE 2

/* Scratch allocator: must return a device pointer to at least `bytes` bytes, 256-byte aligned, valid on
 * `stream` order (a torch.empty(uint8) tensor's data_ptr qualifies), or NULL. */
typedef void* (*gms_alloc_fn)(void* user, int which, size_t bytes);

/* The 13 fields of GaussianRasterizationSettings (renderer/gaussian_renderer/__init__.py:43-57) plus sizes.
 * Matrices/vectors stay on the DEVICE (they are CUDA tensors at the call site). */
typedef struct gms_raster_settings {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    const float* bg;          /* device [3] */
    float scale_modifier;
    const float* viewmatrix;  /* device [16], world_view_transform (transposed W2C), scene/cameras.py:54 */
    const float* projmatrix;  /* device [16], full_proj_transform, scene/cameras.py:56 */
    int32_t sh_degree;        /* active degree 0..3 */
    const float* campos;      /* device [3] */
    int32_t prefiltered;
    int32_t debug;            /* 1: synchronise + check after every launch (stock --debug behaviour) */
    int32_t antialiasing;
} gms_raster_settings;

/* Inputs of GaussianRasterizer.forward (renderer/gaussian_renderer/__init__.py:94-102). Exactly one of
 * shs / colors_precomp and exactly one of (scales, rotations) / cov3D_precomp must be non-NULL. */
typedef struct gms_raster_inputs {
    int32_t P;                   /* number of Gaussians */
    int32_t M;                   /* SH coefficients stored per Gaussian (16 for degree 3); 0 if no shs */
    const float* means3D;        /* [P,3] */
    const float* opacities;      /* [P,1] activated */
    const float* shs;            /* [P,M,3] or NULL */
    const float* colors_precomp; /* [P,3] or NULL */
    const float* scales;         /* [P,3] activated, or NULL */
    const float* rotations;      /* [P,4] (w,x,y,z) normalised, or NULL */
    const float* cov3D_precomp;  /* [P,6] or NULL */
} gms_raster_inputs;

/* Forward outputs (caller-allocated). */
#define GMS_FORWARD_ONLY 1    /* flags bit 0: no backward will follow (inference / no_grad): skip the survivor lists */
typedef struct gms_raster_outputs {
    float* out_color;     /* [3,H,W] */
    int32_t* radii;       /* [P] */
    float* out_invdepth;  /* [1,H,W] */
    int32_t flags;        /* 0, or GMS_FORWARD_ONLY */
} gms_raster_outputs;

/* What forward hands back for backward: scratch base pointers (as returned by the callback) and N. */
typedef struct gms_raster_saved {
    void* geom;
    void* binning;
    void* image;
    int64_t num_rendered;   /* N = number of (tile, Gaussian) duplicates */
    int64_t num_visible;    /* Gaussians with radii > 0 (statistics; may be -1 if not computed) */
    int64_t binning_capacity; /* duplicates the binning region was sized for (== num_rendered on the synchronising call) */
    int32_t flags;          /* bit 0: counting binning layout (point list first; no key arrays); bit 1: per-quad survivor lists
                               of the forward compositing pass follow the point list (consumed by backward); bit 2: the sorted
                               tile keys are 16-bit (tile count <= 65535) -- gms_debug_get_views then reports no key array */
} gms_raster_saved;

/* Gradients produced by backward (caller-allocated; NULL where the corresponding input was NULL). */
typedef struct gms_raster_grads {
    float* dL_dmeans3D;       /* [P,3] */
    float* dL_dmeans2D;       /* [P,3] NDC-scaled screen-space gradient, z = 0 */
    float* dL_dopacities;     /* [P,1] */
    float* dL_dshs;           /* [P,M,3] */
    float* dL_dcolors_precomp;/* [P,3] */
    float* dL_dscales;        /* [P,3] */
    float* dL_drotations;     /* [P,4] */
    float* dL_dcov3D_precomp; /* [P,6] */
    float* dL_dcolors_sh;     /* [P,3] optional, with shs: the clamp-masked colour gradient.  dL/dSH[k][c] = basis_k(dir) * this[c]
                                 (rank 1 per camera), so with it dL_dshs may be NULL: 12 B instead of 192 B per Gaussian
                                 (gms_adam_sh_factored consumes it) */
} gms_raster_grads;

/* ---- rasterizer ------------------------------------------------------------------------------- */

/* Bytes of the per-Gaussian and per-pixel scratch regions (binning depends on N and is requested
 * through the callback once N is known). */
int gms_scratch_bytes(int32_t P, int32_t W, int32_t H, size_t* geom_bytes, size_t* image_bytes);
size_t gms_binning_bytes(int64_t num_rendered, int32_t P);

int gms_rasterize_forward(const gms_raster_settings* settings, const gms_raster_inputs* in,
                          const gms_raster_outputs* out, gms_alloc_fn alloc, void* alloc_user,
                          gms_raster_saved* saved, void* cuda_stream);

/* The same forward WITHOUT the stock pipeline's per-frame host synchronisation ([upstream rasterizer_impl.cu:
 * cudaMemcpy(&num_rendered, ...)]): the caller sizes the binning region for `binning_capacity` duplicates, N is computed
 * and consumed on the device, saved->num_rendered is -1.  `n_host_mapped` (optional) is device-accessible pinned HOST
 * memory [2]: the binning kernel stores N and an overflow flag there, readable later without a sync.  If N exceeds the
 * capacity the frame degrades to the background image with zero gradients (flag = 1) -- grow and re-run.  No allocation,
 * no blocking call: the whole frame can be captured in a CUDA graph. */
int gms_rasterize_forward_nosync(const gms_raster_settings* settings, const gms_raster_inputs* in,
                                 const gms_raster_outputs* out, gms_alloc_fn alloc, void* alloc_user,
                                 gms_raster_saved* saved, int64_t binning_capacity, uint32_t* n_host_mapped,
                                 void* cuda_stream);

/* dL_dout_invdepth may be NULL (train.py never puts a loss on render_pkg["depth"]). */
int gms_rasterize_backward(const gms_raster_settings* settings, const gms_raster_inputs* in,
                           const int32_t* radii, const gms_raster_saved* saved,
                           const float* dL_dout_color /*[3,H,W]*/, const float* dL_dout_invdepth /*[1,H,W]|NULL*/,
                           const gms_raster_grads* grads, void* cuda_stream);

int gms_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present /*[P] bool*/, void* cuda_stream);

/* Read-only views into the scratch regions, for parity tests and statistics (device pointers). */
typedef struct gms_debug_views {
    const float* means2D;        /* packed records [P,12] floats (see gms_debug_unpack for the stock layouts) */
    const float* depths;         /* unused (NULL) */
    const float* cov3D;          /* [P,6] */
    const float* conic_opacity;  /* unused (NULL) */
    const float* rgb;            /* unused (NULL) */
    const uint8_t* clamped;      /* unused (NULL) */
    const uint32_t* tiles_touched; /* [P] */
    const uint32_t* point_list;  /* [N] Gaussian index per duplicate, sorted by (tile, depth bits, index) */
    const uint32_t* tile_keys;   /* [N] tile id per duplicate, sorted */
    const int32_t* ranges;       /* [T,2] */
    const float* final_T;        /* [H,W] */
    const int32_t* n_contrib;    /* [H,W] */
    const float* dgeom;          /* [P,12] after a backward call: per-Gaussian sums the composite backward accumulated --
                                    dL/dmean2D.xy (NDC-scaled), dL/dconic.xyz (stock half convention for xy), dL/d(conic_opacity.w),
                                    dL/drgb.rgb, dL/dinvdepth, 2 unused -- i.e. the input of the preprocess backward */
    const uint32_t* surv;        /* per-quad survivor lists, when the forward wrote them (saved->flags bit 1; else NULL): quad q
                                    of tile t lists, ascending and relative to the tile's list, the positions whose splat blends
                                    into at least one in-image pixel of that quad, at [4 * ranges[t].x + q * n_t, + nsurv[4t+q]),
                                    n_t the length of the tile's list */
    const uint32_t* nsurv;       /* [4T] the length of each of those lists (NULL when there are none) */
} gms_debug_views;
int gms_debug_get_views(const gms_raster_saved* saved, int32_t P, int32_t W, int32_t H, gms_debug_views* views);
/* The per-Gaussian preprocess results live in packed 48-byte records; this unpacks them into the stock
 * layouts (caller-allocated device buffers, any may be NULL): means2D [P,2], depths [P],
 * conic_opacity [P,4], rgb [P,3], clamped [P,3] bytes.  Rows of culled Gaussians are zero. */
int gms_debug_unpack(const gms_raster_saved* saved, int32_t P, const int32_t* radii, float* means2D, float* depths,
                     float* conic_opacity, float* rgb, uint8_t* clamped, void* cuda_stream);

/* ---- mesh -> Gaussian expansion --------------------------------------------------------------- */

#define GMS_ALPHA_RELU 0
#define GMS_ALPHA_SOFTMAX 1

typedef struct gms_expand_args {
    int32_t V, F, K;             /* vertices, faces, splats per face (P = F*K) */
    const float* vertices;       /* [V,3] */
    const int64_t* faces;        /* [F,3] int64 (torch.long), gaussian_mesh_model.py:74 */
    const float* triangles_in;   /* [F,3,3] or NULL: animated path passes transformed triangles directly
                                    (renderer/gaussian_animated_renderer/__init__.py:61-73); then vertices/faces unused */
    const float* alpha_raw;      /* _alpha [F,K,3] */
    const float* scale_raw;      /* _scale [P,1] */
    float eps;                   /* eps_s0 = 1e-8, gaussian_mesh_model.py:43 */
    /* outputs; any may be NULL */
    float* alpha;                /* [F,K,3] normalised barycentrics (pc.alpha) */
    float* triangles;            /* [F,3,3] (pc.triangles) */
    float* xyz;                  /* [P,3] (pc._xyz) */
    float* scaling_log;          /* [P,3] (pc._scaling) */
    float* rotation_raw;         /* [P,4] (pc._rotation) */
    float* scaling_act;          /* [P,3] = exp(_scaling)        (get_scaling, fused E4) */
    float* rotation_act;         /* [P,4] = normalize(_rotation) (get_rotation, fused E4) */
    int32_t alpha_activation;    /* barycentric weights from _alpha: GMS_ALPHA_RELU (0) relu + 1e-8, normalised (gs_mesh,
                                    gaussian_mesh_model.py:166-167); GMS_ALPHA_SOFTMAX (1) softmax over the three
                                    (gs_flame, gaussian_flame_model.py:34,195); anything else is GMS_E_ARG */
} gms_expand_args;

int gms_expand_forward(const gms_expand_args* a, void* cuda_stream);

typedef struct gms_expand_grads {
    /* incoming (any may be NULL = zero) */
    const float* dL_dxyz;          /* [P,3] */
    const float* dL_dscaling_log;  /* [P,3] */
    const float* dL_drotation_raw; /* [P,4] */
    const float* dL_dscaling_act;  /* [P,3] gradient w.r.t. exp(_scaling) */
    const float* dL_drotation_act; /* [P,4] gradient w.r.t. normalize(_rotation) */
    /* outgoing */
    float* dL_dvertices;           /* [V,3] ACCUMULATED with atomics: caller zero-fills; NULL if triangles_in */
    float* dL_dtriangles;          /* [F,3,3] written (NULL allowed) */
    float* dL_dalpha_raw;          /* [F,K,3] */
    float* dL_dscale_raw;          /* [P,1] */
} gms_expand_grads;

int gms_expand_backward(const gms_expand_args* a, const gms_expand_grads* g, void* cuda_stream);

/* gs_points pseudo-mesh path: one triangle per Gaussian -> (xyz = v1, 2 log-scales, quaternion).  Replaces
 * PointsGaussianModel.prepare_scaling_rot (games/flat_splatting/scene/points_gaussian_model.py:61-104) as called per
 * frame by renderer/gaussian_points_animated_renderer/__init__.py:61-66.  Forward only (render scripts, no_grad). */
typedef struct gms_points_args {
    int32_t P;
    const float* triangles;      /* [P,3,3] */
    float eps;                   /* 1e-8 */
    float* xyz;                  /* [P,3] = triangles[:,0]            (any output may be NULL) */
    float* scaling_log;          /* [P,2] (pc._scaling) */
    float* rotation_raw;         /* [P,4] (pc._rotation) */
    float* scaling_act;          /* [P,3] = (eps, exp(_scaling))      (get_scaling) */
    float* rotation_act;         /* [P,4] = normalize(_rotation)      (get_rotation) */
} gms_points_args;
int gms_points_expand_forward(const gms_points_args* a, void* cuda_stream);

/* gs_points, the other direction: every flat Gaussian -> its pseudo-mesh triangle (v1 = xyz, v2/v3 = xyz + s*axis, the
 * longer arm first).  Replaces PointsGaussianModel.prepare_vertices (games/flat_splatting/scene/points_gaussian_model.py:
 * 28-59, with get_scaling :106-109 and build_rotation utils/general_utils.py:158-179), run once when a trained gs_flat
 * model is loaded for editing (scripts/render_points_time_animated.py).  Forward only. */
typedef struct gms_points_vertices_args {
    int32_t P;
    const float* xyz;            /* [P,3]  pc._xyz */
    const float* scaling_log;    /* [P,scaling_cols]  pc._scaling; the LAST two columns are the in-plane log-scales */
    int32_t scaling_cols;        /* 2 (gs_points) or 3 (a gs_flat checkpoint) */
    const float* rotation_raw;   /* [P,4]  pc._rotation (w,x,y,z), not normalised */
    float* triangles;            /* out [P,3,3] */
} gms_points_vertices_args;
int gms_points_prepare_vertices(const gms_points_vertices_args* a, void* cuda_stream);

/* ---- training-step glue on the same stream (SURVEY.md section 8(f) ranks 1-2: the callers either side of the path) ---- */

/* L = (1-lambda)*L1 + lambda*(1-SSIM) and dL/dimg in two launches.  Replaces utils/loss_utils.py:17-64 as used by
 * train.py:105-108 (5 grouped conv2d forward + 5 backward + ~30 elementwise launches per frame). */
typedef struct gms_loss_args {
    int32_t C, H, W;
    const float* img;        /* [C,H,W] rendered image */
    const float* gt;         /* [C,H,W] ground truth */
    float lambda_dssim;      /* 0.2, arguments/__init__.py:86 */
    const float* dL_dloss;   /* device scalar upstream gradient, or NULL for 1 */
    float* loss;             /* device [3]: loss, L1 mean, SSIM mean */
    float* dL_dimg;          /* [C,H,W] or NULL (forward only) */
    void* scratch;           /* gms_loss_scratch_bytes() bytes */
    size_t scratch_bytes;
} gms_loss_args;
int gms_loss_scratch_bytes(int32_t C, int32_t H, int32_t W, size_t* bytes);
int gms_l1_ssim_loss(const gms_loss_args* a, void* cuda_stream);

/* torch.optim.Adam(groups, eps=1e-15) of gaussian_mesh_model.py:171-183 (train.py:146-148) over ONE flat fp32
 * parameter buffer, one launch; consumes and (optionally, fully or only a leading range) zeroes the gradient in the same pass.
 * Segment i covers flat indices [seg_end[i-1], seg_end[i]); lr = lr0[i], or -- when period[i] > 0 --
 * lr0[i] where ((index - segment start) / inner[i]) % period[i] == 0 and lr1[i] elsewhere (DC vs rest SH). */
typedef struct gms_adam_args {
    int64_t n;               /* elements this call updates */
    int64_t offset;          /* flat index of element 0 (sharded optimizer: each rank updates [offset, offset+n)); 0 otherwise */
    float* p; float* g; float* m; float* v;   /* pointers to element `offset` of the respective flat buffers */
    int32_t nseg;
    int64_t seg_end[8];
    double lr0[8]; double lr1[8];   /* doubles, like torch's Python-float hyper-parameters: lr / (1 - beta1^t), 1 - beta */
    int32_t inner[8]; int32_t period[8];
    double beta1, beta2, eps;       /* and sqrt(1 - beta2^t) are formed in double and rounded to fp32 once */
    int32_t step;            /* 1-based step count (bias correction) */
    int32_t zero_grad;       /* 0: leave g; 1: zero every consumed element; 2: zero only flat indices < zero_end */
    int64_t zero_end;        /* (mode 2) e.g. the end of the vertices segment when every other gradient is overwritten
                                by the next frame (gms_train_frame) */
} gms_adam_args;
int gms_adam_step(const gms_adam_args* a, void* cuda_stream);

/* The Adam step gms_train_frame can apply to the packed SH parameter inside its preprocess backward (gms_frame_args.sh_adam):
 * bit for bit what gms_adam_sh_factored does with one slot (R = 1, grad_scale 1) holding this frame's d_color_sh, without
 * the slot's round trip through memory or a second read of the parameter.  One camera per step only (data parallel: exchange
 * the colour gradients through d_color_sh instead). */
typedef struct gms_sh_adam {
    float* m; float* v;         /* [P,16,3] Adam moments of `features` */
    double lr_dc, lr_rest, beta1, beta2, eps;
    int32_t step;               /* 1-based step count (bias correction) */
} gms_sh_adam;

/* One gs_mesh training frame in ONE call (train.py:100-108 + :154-157 of the reference: render + loss + backward +
 * re-expansion), all launches on `cuda_stream`, no Python / autograd in between:
 *   expansion fwd (activated scales/rotations) -> sigmoid(opacity) -> rasterizer fwd -> L1+SSIM -> rasterizer bwd ->
 *   sigmoid bwd -> expansion bwd.
 * Model tensors are the RAW parameters; gradients are written (d_vertices: accumulated with atomics, keep it zeroed)
 * into caller buffers, e.g. views of the flat gradient buffer gms_adam_step / the NCCL exchange operate on.
 * `workspace` holds the per-frame intermediates (gms_frame_workspace_bytes); the rasterizer's scratch still comes
 * through the allocation callback. */
/* One mesh of a gs_multi_mesh scene whose meshes use different splat counts (train.py --num_splats a b ...;
 * games/multi_mesh_splatting/scene/gaussian_multi_mesh_model.py:99-199).  With n_segments > 0 in gms_frame_args /
 * gms_render_args:
 *   - `faces` holds the meshes' faces one after another, already re-indexed into the one `vertices` array;
 *   - F = sum F_i and K = 0; every F_i >= 1 and K_i >= 1; P = sum F_i * K_i must fit int32;
 *   - mesh i's Gaussians are the contiguous rows [P_i, P_i + F_i*K_i) of every per-Gaussian array, P_i = sum_{j<i} F_j*K_j
 *     (the reference's torch.cat order): alpha_raw [P,3] holds mesh i's [F_i,K_i,3] at row P_i, scale_raw is [P,1].
 * The expansion runs once per mesh (forward and backward: one launch each per mesh); everything after it runs once over all
 * P Gaussians.  Anything else is GMS_E_ARG, returned before any launch. */
typedef struct gms_mesh_segment {
    int32_t F, K;
} gms_mesh_segment;

typedef struct gms_frame_args {
    int32_t V, F, K, M;
    const float* vertices; const int64_t* faces; const float* alpha_raw; const float* scale_raw;
    const float* features;      /* [P,M,3] packed SH (get_features) */
    const float* opacity_raw;   /* [P,1] logits */
    float eps;                  /* eps_s0 */
    float* d_vertices; float* d_alpha_raw; float* d_scale_raw; float* d_features; float* d_opacity_raw;
    gms_raster_settings settings;
    const float* gt;            /* [3,H,W] */
    float lambda_dssim;
    float* loss;                /* device [3]: loss, L1, SSIM */
    void* workspace; size_t workspace_bytes;
    int64_t* num_rendered;      /* host, optional (-1 on the sync-free path) */
    int64_t binning_capacity;   /* > 0: sync-free frame (gms_rasterize_forward_nosync semantics); 0: stock-style, one 4-byte D2H */
    uint32_t* n_host_mapped;    /* optional mapped pinned host [2]: N, overflow flag */
    float* d_color_sh;          /* optional [3P + 3]: factored SH gradient (dL_dcolors_sh) followed by this frame's camera centre;
                                   then d_features may be NULL and no SH gradient rows are written */
    void* event_sh_ready;       /* optional cudaEvent_t recorded right after the preprocess backward: d_color_sh (or d_features) is
                                   final from there on, so a data-parallel caller can start exchanging it on another stream while the
                                   opacity / expansion backward still runs */
    void* event_loss_ready;     /* optional cudaEvent_t recorded right after the loss kernels (about 40 % into the frame): a caller that
                                   logs the loss every step copies it to the host from another stream and can queue the next
                                   frame while this one's backward pass still runs */
    const gms_sh_adam* sh_adam; /* optional: the frame also takes the Adam step of `features` (updated in place, M = 16) with
                                   this frame's SH gradient; then d_features and d_color_sh may be NULL */
    const gms_mesh_segment* segments;   /* HOST [n_segments] or NULL: gs_multi_mesh with a K per mesh (see gms_mesh_segment) */
    int32_t n_segments;                 /* 0: one mesh of F faces x K splats, P = F*K */
    uint32_t anomaly_stages;            /* bit (1 << GMS_ANOMALY_*) per stage: LOSS, COMPOSITE_BWD, PREPROCESS_BWD, EXPAND_BWD */
    uint64_t* anomaly;                  /* optional device record of gms_nan_scan: the outputs of every backward stage selected in
                                           anomaly_stages are scanned for NaN right after that stage (see "anomaly detection");
                                           NULL: no scan, the frame's launches are unchanged.  Not with sh_adam (GMS_E_ARG) */
    int32_t alpha_activation;           /* as gms_expand_args.alpha_activation (every segment): 0 gs_mesh, 1 gs_flame; the trailing
                                           field, as in gms_render_args and gms_expand_args */
} gms_frame_args;
size_t gms_frame_workspace_bytes(int32_t P, int32_t W, int32_t H);
/* Device pointers into a frame workspace (valid after gms_train_frame): this step's expansion outputs and images. */
typedef struct gms_frame_view {
    const float* xyz; const float* scales; const float* rotations; const float* opacities; const int32_t* radii;
    const float* image; const float* invdepth;
} gms_frame_view;
int gms_frame_views(void* workspace, int32_t P, int32_t W, int32_t H, gms_frame_view* v);

/* Adam step of the packed SH parameter [P,16,3] with its gradient rebuilt from FACTORS instead of read from memory:
 *   dL/dSH_i[k][c] = grad_scale * sum_r basis_k(normalize(xyz_i - campos_r)) * dcolor_r[i][c],   r = 0..R-1
 * `exchange` holds R slots of `slot_floats` floats, slot r = [3P colour gradients of frame r | its camera centre (3) | pad]
 * (what gms_train_frame writes through d_color_sh).  Data parallel: the slots are all-gathered (12 B per Gaussian and
 * rank instead of a 192 B reduce-scatter + all-gather), every rank runs this kernel on all Gaussians (replicated moments),
 * so no parameter all-gather is needed either.  Learning rates / bias correction as in gms_adam_step (DC coefficient:
 * lr_dc, the other 15: lr_rest; arguments_games/__init__.py:17-30). */
typedef struct gms_adam_sh_args {
    int32_t P, M, sh_degree, R;
    const float* xyz;          /* [P,3] Gaussian centres of this step (gms_frame_views) */
    const float* exchange;     /* [R, slot_floats] */
    int64_t slot_floats;
    float grad_scale;          /* 1/R */
    float* p; float* m; float* v;
    double lr_dc, lr_rest, beta1, beta2, eps;
    int32_t step;
} gms_adam_sh_args;
int gms_adam_sh_factored(const gms_adam_sh_args* a, void* cuda_stream);
int gms_train_frame(const gms_frame_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* ---- rendering and evaluating views ------------------------------------------------------------- */

/* One gs_mesh render in ONE call: the forward half of gms_train_frame (expansion fwd with activated scales / rotations ->
 * sigmoid(opacity) inside the preprocess -> rasterizer fwd), as a forward-only frame (GMS_FORWARD_ONLY: the binning region
 * holds the point list only).  Replaces the per-view render of scripts/render.py:25-36 and of the animated sweep,
 * renderer/gaussian_animated_renderer/__init__.py:61-112 (for scripts/render_time_animated.py the caller moves `vertices`
 * first, as its :82-84 does).  num_rendered / binning_capacity / n_host_mapped: exactly as in gms_frame_args -- a capacity
 * of 0 reads N back once (one host synchronisation), a capacity > 0 never synchronises and an overflow (N > capacity)
 * renders the background with zero inverse depth. */
typedef struct gms_render_args {
    int32_t V, F, K, M;
    const float* vertices; const int64_t* faces; const float* alpha_raw; const float* scale_raw;
    const float* features;      /* [P,M,3] packed SH (get_features) */
    const float* opacity_raw;   /* [P,1] logits */
    float eps;                  /* eps_s0 */
    gms_raster_settings settings;
    float* image;               /* out [3,H,W] */
    float* invdepth;            /* out [1,H,W] */
    int32_t* radii;             /* out [P] */
    void* workspace; size_t workspace_bytes;   /* gms_render_workspace_bytes: the expansion outputs and opacities only */
    int64_t* num_rendered;      /* host, optional (-1 on the sync-free path) */
    int64_t binning_capacity;
    uint32_t* n_host_mapped;    /* optional mapped pinned host [2]: N, overflow flag */
    const gms_mesh_segment* segments;   /* HOST [n_segments] or NULL: as in gms_frame_args */
    int32_t n_segments;
    int32_t alpha_activation;           /* as gms_expand_args.alpha_activation */
} gms_render_args;
size_t gms_render_workspace_bytes(int32_t P, int32_t W, int32_t H);
int gms_render_frame(const gms_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* One gs_flame render of a trained checkpoint in ONE call, the protocol of scripts/render_flame.py
 * (renderer/flame_gaussian_renderer/__init__.py:59-80): xyz = alpha [F,K,3] (the ACTIVATED weights flame_params.pt stores)
 * times vertices[faces] of the driving pose; scales = exp(_scaling) and rotations = normalize(_rotation) from the
 * checkpoint's rows -- they do not follow the pose, as in the reference; sigmoid(opacity) inside the preprocess.  One
 * activation launch, then the rasterizer forward of gms_render_frame.  Capacity semantics, outputs and validation as in
 * gms_render_args; P = F*K; rotation_raw must be 16-byte aligned. */
typedef struct gms_flame_render_args {
    int32_t V, F, K, M;
    const float* vertices;      /* [V,3] driving pose */
    const int64_t* faces;       /* [F,3] */
    const float* alpha;         /* [F,K,3] activated barycentric weights */
    const float* scaling_log;   /* [P,3] _scaling of the checkpoint */
    const float* rotation_raw;  /* [P,4] _rotation of the checkpoint */
    const float* features;      /* [P,M,3] packed SH */
    const float* opacity_raw;   /* [P,1] logits */
    gms_raster_settings settings;
    float* image; float* invdepth; int32_t* radii;
    void* workspace; size_t workspace_bytes;   /* gms_flame_render_workspace_bytes */
    int64_t* num_rendered;
    int64_t binning_capacity;
    uint32_t* n_host_mapped;
} gms_flame_render_args;
size_t gms_flame_render_workspace_bytes(int32_t P, int32_t W, int32_t H);
int gms_flame_render_frame(const gms_flame_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* One gs_points (pseudo-mesh) render in ONE call: the pseudo-mesh expansion (gms_points_expand_forward with activated outputs:
 * xyz = v1, scaling (eps, exp(log s2), exp(log s3)), normalised quaternion) -> sigmoid(opacity) inside the preprocess ->
 * rasterizer fwd, as a forward-only frame (GMS_FORWARD_ONLY: the binning region holds the point list only).  Replaces the
 * per-view render of renderer/gaussian_points_animated_renderer/__init__.py:21-114 (prepare_scaling_rot(triangles), the
 * getters and GaussianRasterizer) as scripts/render_points_time_animated.py, scripts/render_from_object.py and
 * scripts/render.py --gs_type gs_points call it; the caller transforms `triangles` first, as those scripts do.  Unlike the
 * reference, nothing of the model is overwritten.  num_rendered / binning_capacity / n_host_mapped: exactly as in
 * gms_render_args. */
typedef struct gms_points_render_args {
    int32_t P, M;
    const float* triangles;     /* [P,3,3] pseudo-mesh triangles of this frame */
    const float* features;      /* [P,M,3] packed SH (get_features) */
    const float* opacity_raw;   /* [P,1] logits */
    float eps;                  /* eps_s0 = prepare_scaling_rot's eps, 1e-8 */
    gms_raster_settings settings;
    float* image;               /* out [3,H,W] */
    float* invdepth;            /* out [1,H,W] */
    int32_t* radii;             /* out [P] */
    void* workspace; size_t workspace_bytes;   /* gms_points_render_workspace_bytes: the expansion outputs and opacities only */
    int64_t* num_rendered;      /* host, optional (-1 on the sync-free path) */
    int64_t binning_capacity;
    uint32_t* n_host_mapped;    /* optional mapped pinned host [2]: N, overflow flag */
} gms_points_render_args;
size_t gms_points_render_workspace_bytes(int32_t P, int32_t W, int32_t H);
int gms_points_render_frame(const gms_points_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* Mesh-driven pseudo-mesh editing (scripts/edit_pseudomesh_based_on_estimated_mesh.py:14-94, README "Pseudomesh/Triangle
 * Soup and modifications"): every pseudo-triangle tracks the nearest face of a driving mesh, so moving that mesh's vertices
 * moves the Gaussians.
 *
 * Binding (:25-54), once per pseudo-mesh and rest-pose mesh:
 *   - face i = the non-degenerate face whose centroid ((v0 + v1) + v2) / 3 (fp32) is nearest to the pseudo-triangle's
 *     centroid, by the squared distance in double (dx*dx + dy*dy) + dz*dz, the lowest index on an exact tie.  This is the
 *     reference's sklearn KDTree query except at exact ties.  A face is degenerate when |v2 - v1|, |v3 - v1| or
 *     |cross(v2 - v1, v3 - v1)| is exactly 0 in fp32; the reference would bind to it and produce NaN.
 *   - coeffs[i][j] = the solution of [n|e1|e2] c = w_j - v1 for pseudo-vertex w_j, in double, rounded to fp32, with the skewed
 *     frame n = normalise(cross(v2 - v1, v3 - v1)), e1 = normalise(v2 - v1), e2 = normalise(v3 - v1) of face i.
 * Every face index must lie in [0, V) (not checked here: the caller's responsibility, as for gms_expand_args).  The call
 * synchronises the stream once, to count the degenerate faces.  GMS_E_ARG: a null pointer, P < 0, F < 1, V < 1, too
 * little scratch, or every face degenerate (n_degenerate is still written). */
typedef struct gms_pseudomesh_bind_args {
    int32_t P;
    const float* triangles;     /* [P,3,3] pseudo-mesh (this and the outputs may be NULL when P == 0) */
    int32_t V, F;
    const float* vertices;      /* [V,3] rest pose of the driving mesh */
    const int64_t* faces;       /* [F,3] */
    int32_t* face;              /* out [P] bound face */
    float* coeffs;              /* out [P,3,3] coefficients of (n, e1, e2) per pseudo-vertex */
    int32_t* n_degenerate;      /* out, host: degenerate faces of the mesh (never bound) */
    void* scratch; size_t scratch_bytes;   /* gms_pseudomesh_bind_scratch_bytes(F) */
} gms_pseudomesh_bind_args;
size_t gms_pseudomesh_bind_scratch_bytes(int32_t F);
int gms_pseudomesh_bind(const gms_pseudomesh_bind_args* a, void* cuda_stream);

/* Re-posing a binding on a pose of the same mesh (same faces; :58-82): w_j = ((v1' + c_j0 n') + c_j1 e1') + c_j2 e2' with the
 * frame of the bound face in that pose.  A face degenerate in that pose gives non-finite triangles, as in the reference.
 * Face indices: as in gms_pseudomesh_bind_args. */
typedef struct gms_pseudomesh_repose_args {
    int32_t P;
    const int32_t* face;        /* [P] from gms_pseudomesh_bind, each in [0, F) */
    const float* coeffs;        /* [P,3,3] */
    int32_t V, F;
    const float* vertices;      /* [V,3] driving pose */
    const int64_t* faces;       /* [F,3] */
    float* triangles;           /* out [P,3,3] (unused by gms_bound_points_render_frame) */
} gms_pseudomesh_repose_args;
int gms_pseudomesh_repose(const gms_pseudomesh_repose_args* a, void* cuda_stream);

/* One gs_points render of a bound pseudo-mesh in a driving pose, in ONE call: the re-pose and the pseudo-mesh expansion of
 * gms_points_render_frame fused in one kernel (the triangles are never written), then the same forward-only rasterizer
 * forward.  Gaussians whose bound face is degenerate in this pose are culled (radius 0, no tile).  Workspace, num_rendered /
 * binning_capacity / n_host_mapped: exactly as in gms_points_render_args. */
typedef struct gms_bound_points_render_args {
    int32_t P, M;
    const int32_t* face;        /* [P] binding */
    const float* coeffs;        /* [P,3,3] binding */
    int32_t V, F;
    const float* vertices;      /* [V,3] driving pose of this frame */
    const int64_t* faces;       /* [F,3], each index in [0, V) */
    const float* features;      /* [P,M,3] packed SH (get_features) */
    const float* opacity_raw;   /* [P,1] logits */
    float eps;                  /* eps_s0 = prepare_scaling_rot's eps, 1e-8 */
    gms_raster_settings settings;
    float* image;               /* out [3,H,W] */
    float* invdepth;            /* out [1,H,W] */
    int32_t* radii;             /* out [P] */
    void* workspace; size_t workspace_bytes;   /* gms_bound_points_render_workspace_bytes */
    int64_t* num_rendered;      /* host, optional (-1 on the sync-free path) */
    int64_t binning_capacity;
    uint32_t* n_host_mapped;    /* optional mapped pinned host [2]: N, overflow flag */
} gms_bound_points_render_args;
size_t gms_bound_points_render_workspace_bytes(int32_t P, int32_t W, int32_t H);
int gms_bound_points_render_frame(const gms_bound_points_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* ---- free Gaussians: gs and gs_flat ----------------------------------------------------------------- */

/* One gs / gs_flat training frame in ONE call: gms_train_frame with the mesh expansion replaced by the per-Gaussian
 * activation of scene/gaussian_model.py:95-101 (games/flat_splatting/scene/flat_gaussian_model.py:32-35 for gs_flat):
 *   scales = exp(scaling_raw) (gs, scale_cols 3) or (eps, exp(scaling_raw[:,0]), exp(scaling_raw[:,1])) (gs_flat, scale_cols 2),
 *   rotations = rotation_raw / max(|rotation_raw|, 1e-12); xyz is the raw parameter itself.
 * -> sigmoid(opacity) -> rasterizer fwd -> L1+SSIM -> rasterizer bwd -> raw gradients of scaling (none for the eps column)
 * and rotation.  d_xyz receives dL/dxyz directly.  With accum / denom ([P] float) the same pass adds the densification
 * statistics of add_densification_stats (scene/gaussian_model.py:416-418): accum += |dL/dmeans2D.xy|, denom += 1 where
 * radii > 0 -- except on an overflowed sync-free frame, which adds nothing.  num_rendered / binning_capacity / n_host_mapped /
 * event_loss_ready / sh_adam: as in gms_frame_args; the workspace is gms_frame_workspace_bytes(P, W, H).  As many launches as
 * gms_train_frame.  Quaternion rows move as float4: rotation_raw and d_rotation_raw must be 16-byte aligned. */
typedef struct gms_free_frame_args {
    int32_t P, M;
    int32_t scale_cols;         /* 3 (gs) or 2 (gs_flat) */
    const float* xyz;           /* [P,3] _xyz */
    const float* scaling_raw;   /* [P,scale_cols] _scaling */
    const float* rotation_raw;  /* [P,4] _rotation, 16-byte aligned (GMS_E_ARG otherwise) */
    const float* features;      /* [P,M,3] packed SH */
    const float* opacity_raw;   /* [P,1] logits */
    float eps;                  /* gs_flat eps_s0 = 1e-8 (unused for gs) */
    float* d_xyz; float* d_scaling_raw; float* d_rotation_raw /* 16-byte aligned */; float* d_features; float* d_opacity_raw;
    float* accum; float* denom; /* optional [P]: xyz_gradient_accum, denom (both or neither) */
    gms_raster_settings settings;
    const float* gt;            /* [3,H,W] */
    float lambda_dssim;
    float* loss;                /* device [3]: loss, L1, SSIM */
    void* workspace; size_t workspace_bytes;
    int64_t* num_rendered;
    int64_t binning_capacity;
    uint32_t* n_host_mapped;
    void* event_loss_ready;
    const gms_sh_adam* sh_adam; /* optional: fused Adam step of `features` (M = 16); then d_features may be NULL */
    uint64_t* anomaly;          /* as in gms_frame_args; the stages are LOSS, COMPOSITE_BWD, PREPROCESS_BWD, ACTIVATION_BWD */
    uint32_t anomaly_stages;
} gms_free_frame_args;
int gms_free_train_frame(const gms_free_frame_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* The forward half of gms_free_train_frame as a forward-only frame (GMS_FORWARD_ONLY), with gms_render_frame's capacity
 * semantics; the workspace is gms_render_workspace_bytes(P, W, H). */
typedef struct gms_free_render_args {
    int32_t P, M, scale_cols;
    const float* xyz; const float* scaling_raw; const float* rotation_raw /* 16-byte aligned */; const float* features;
    const float* opacity_raw;
    float eps;
    gms_raster_settings settings;
    float* image;               /* out [3,H,W] */
    float* invdepth;            /* out [1,H,W] */
    int32_t* radii;             /* out [P] */
    void* workspace; size_t workspace_bytes;
    int64_t* num_rendered;
    int64_t binning_capacity;
    uint32_t* n_host_mapped;
} gms_free_render_args;
int gms_free_render_frame(const gms_free_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* densify_and_prune (scene/gaussian_model.py:360-414; flat_gaussian_model.py:62-88) in two calls.
 * gms_densify_plan decides every row's fate from grads = accum / denom (0 / 0 -> 0) and S = max(get_scaling):
 *   clone  grads >= grad_threshold and S <= split_scale (percent_dense * extent)
 *   split  grads >= grad_threshold and S >  split_scale (the original is removed; two children replace it)
 *   prune  sigmoid(opacity) < min_opacity, or (max_world_scale > 0) get_scaling.max > max_world_scale (0.1 * extent, the
 *          reference's big_points_ws when max_screen_size is set) -- for originals, clones, and split children (judged by
 *          their own scaling).  The screen-space prune never fires in the reference (max_radii2D is all zeros there) and
 *          is not offered.
 * A scan gives every surviving row its position in the reference's order: kept originals, clones, split copy 0 of every
 * split row, split copy 1.  The call synchronises the stream ONCE and writes result[5] (host): the new P, the kept
 * originals, the surviving clones, the surviving split pairs (each gives two rows) and the pruned rows.  P = 0 is valid. */
#define GMS_FATE_CLONE 1
#define GMS_FATE_SPLIT 2
#define GMS_FATE_PRUNE 4            /* the row (and its clone) fails the prune */
#define GMS_FATE_PRUNE_CHILDREN 8   /* its split children fail the prune */
typedef struct gms_densify_plan_args {
    int32_t P, scale_cols;
    const float* accum; const float* denom;   /* [P] */
    const float* scaling_raw;                 /* [P,scale_cols] */
    const float* opacity_raw;                 /* [P,1] */
    float eps;                                /* gs_flat eps_s0 */
    float grad_threshold, split_scale, min_opacity, max_world_scale;
    uint8_t* fate;                            /* optional out [P]: GMS_FATE_* bits */
    void* scratch; size_t scratch_bytes;      /* gms_densify_scratch_bytes(P); gms_densify_apply reads the plan from it */
    int32_t* result;                          /* host [5] */
} gms_densify_plan_args;
size_t gms_densify_scratch_bytes(int32_t P);
int gms_densify_plan(const gms_densify_plan_args* a, void* cuda_stream);

/* One set of per-Gaussian rows: the raw parameters, or one Adam moment of each of them. */
typedef struct gms_free_set {
    float* xyz;       /* [P,3] */
    float* scaling;   /* [P,scale_cols] */
    float* rotation;  /* [P,4] */
    float* opacity;   /* [P,1] */
    float* features;  /* [P,M,3] */
} gms_free_set;

/* Builds the densified set the plan in `scratch` describes into caller-allocated rows of the new size (result[0] of that
 * plan): parameters and both Adam moments (src/dst[0] parameters, [1] exp_avg, [2] exp_avg_sq).  Kept originals carry
 * their moments, clones and split children get zero moments.  Split child c of row i: xyz = R(q_i) (get_scaling_i *
 * normals[i][c]) + xyz_i, scaling = log(get_scaling_i / 1.6) (columns [1,2] of it for gs_flat); normals [P,2,3] are
 * standard-normal draws.  Sources are read only; destinations may not overlap them. */
typedef struct gms_densify_apply_args {
    int32_t P, new_P, scale_cols, M;
    float eps;
    const void* scratch; size_t scratch_bytes;   /* as left by gms_densify_plan for the same P */
    const int32_t* result;                       /* host [5], gms_densify_plan's */
    const float* normals;                        /* [P,2,3] */
    gms_free_set src[3];
    gms_free_set dst[3];
} gms_densify_apply_args;
int gms_densify_apply(const gms_densify_apply_args* a, void* cuda_stream);

/* ---- point-cloud initialisation ------------------------------------------------------------------ */

/* simple-knn's distCUDA2 (the initial scales of create_from_pcd, scene/gaussian_model.py:124-147): for every point, the mean
 * squared distance to its three nearest OTHER points, exactly.
 *   d(q,p)   = (dx*dx + dy*dy) + dz*dz, dx = q.x - p.x, each operation one round-to-nearest fp32 op (no FMA)
 *   b0 <= b1 <= b2: the three smallest d(points[i], points[j]) over j != i; tied values (duplicate points at 0) count
 *   separately
 *   dist2[i] = ((b0 + b1) + b2) / 3, round-to-nearest
 * The result depends only on the multiset of distances: two calls give the same bits, whatever the launch order.  The search
 * prunes with Morton-ordered boxes of GMS_KNN_BOX points whose lower bounds round as d does, so pruning is exact (DESIGN.md
 * 4.4).  P = 0 is a no-op; 1 <= P <= 3 (no three neighbours), a null pointer or too little scratch is GMS_E_ARG.  No host
 * synchronisation. */
#define GMS_KNN_BOX 64
typedef struct gms_knn_args {
    int32_t P;
    const float* points;                   /* [P,3] device, every coordinate finite (not checked here) */
    float* dist2;                          /* out [P] */
    void* scratch; size_t scratch_bytes;   /* gms_knn_scratch_bytes(P) */
} gms_knn_args;
size_t gms_knn_scratch_bytes(int32_t P);
int gms_knn_dist2(const gms_knn_args* a, void* cuda_stream);

/* ---- the editing mesh of a pseudo-mesh (scripts/create_dummy_mesh.py) ----------------------------- */

/* open3d's CreateFromPointCloudAlphaShape for finite float32 points [P,3], every geometric quantity in float64 (DESIGN.md 4.11).
 *   Exact duplicates: a point equal to a point of lower index takes no part (the written positions are the same either way).
 *   Triangle (a < b < c) is output iff it is a face of the Delaunay tetrahedralization of the remaining points and exactly
 *   one of its (one or two) incident tetrahedra has circumradius <= alpha.  For points in general position this is open3d's
 *   triangle set.  Tie rule under degeneracy: with w = (b-a) x (c-a), circumcentre c_f and tau_p = (|p-c_f|^2 - r_f^2) /
 *   (2 w.(p-c_f)), T+ = min tau over w.(p-c_f) > 0 and T- = max over < 0, the face is Delaunay iff T- < T+ strictly and no
 *   point with w.(p-c_f) == 0 lies strictly inside the circumcircle; a side is kept iff r_f^2 + |w|^2 tau^2 <= alpha^2.
 *   Collinear triples are never output.  This need not match Qhull's choice for cospherical or coplanar points.
 *   Order: vertices are the referenced points in ascending original index (index[V], int64); faces[F,3] (int64, rows of the
 *   vertex list) have ascending vertex indices and are in lexicographic order.
 * The call sizes its memory through alloc(user, which, bytes) with which = GMS_ALPHA_BUF_*: SCRATCH (P-sized), LISTS (the
 * neighbour lists, known after the first of two host synchronisations), FACES ([F,3] int64) and INDEX ([V] int64), the last
 * two after the second and only when non-empty.  The caller owns what it returned and reads faces / index from it.
 * GMS_E_ARG before any launch: a null pointer, P < 0, P = INT32_MAX, alpha <= 0 or not finite; after the first
 * synchronisation when the 2-alpha lists hold 2^31 entries or more.  GMS_E_ALLOC when alloc returns NULL.  P = 0 gives
 * F = V = 0 without a launch.  Runs on the caller's stream and returns after the last launch is enqueued. */
#define GMS_ALPHA_BUF_SCRATCH 0
#define GMS_ALPHA_BUF_LISTS 1
#define GMS_ALPHA_BUF_FACES 2
#define GMS_ALPHA_BUF_INDEX 3
#define GMS_ALPHA_LIST_CAP 256     /* 3-alpha list entries staged in shared memory per point; longer lists are read from global */
typedef struct gms_alpha_shape_args {
    int32_t P;
    const float* points;        /* [P,3] device, every coordinate finite (not checked here) */
    double alpha;
    int64_t* n_faces;           /* out, host: F */
    int64_t* n_vertices;        /* out, host: V */
} gms_alpha_shape_args;
int gms_alpha_shape(const gms_alpha_shape_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream);

/* open3d's EstimateNormals(KDTreeSearchParamHybrid(radius, max_nn)) with a stated sign.  For every point: the min(max_nn, k)
 * nearest points by (float64 squared distance, index) with distance <= radius, the point itself and its duplicates
 * included; the unit eigenvector of the smallest eigenvalue of their mean-centred float64 covariance (cyclic Jacobi), or
 * (0,0,1) when k < 3.  Sign: n.(x - mean of all P points) >= 0; when that is exactly 0 the largest-magnitude component (the
 * first of equals) is positive.  GMS_E_ARG before any launch: a null pointer, P < 0, radius <= 0 or not finite,
 * max_nn outside 1..GMS_NORMALS_MAX_NN, too little scratch.  P = 0 is a no-op.  Caller's stream, no host synchronisation. */
#define GMS_NORMALS_MAX_NN 64
typedef struct gms_normals_args {
    int32_t P;
    const float* points;                   /* [P,3] device, finite */
    double radius;
    int32_t max_nn;
    float* normals;                        /* out [P,3] */
    void* scratch; size_t scratch_bytes;   /* gms_normals_scratch_bytes(P) */
} gms_normals_args;
size_t gms_normals_scratch_bytes(int32_t P);
int gms_estimate_normals(const gms_normals_args* a, void* cuda_stream);

/* ---- FLAME's vertex model (gs_flame) ----------------------------------------------------------- */

/* FLAME.forward's vertices (games/flame_splatting/FLAME/FLAME.py:204-248 with smplx.lbs.lbs, landmarks left out) followed by
 * transform_vertices_function (games/flame_splatting/scene/dataset_readers.py:40-45), for one frame:
 *   betas    = [shape, expression] (the active columns; the reference's zero-padded ones contribute nothing)
 *   v_shaped = v_template + shapedirs^T betas;  J = J_regressor . v_shaped
 *   R_j      = batch_rodrigues(full_pose_j), full_pose = [pose[:3], neck_pose, pose[3:], eye_pose = 0]
 *   v_posed  = v_shaped + ((R_1..4 - I) flattened) . posedirs
 *   A_j      = batch_rigid_transform's relative transforms over `parents`
 *   o        = (sum_j lbs_weights[v,j] A_j) [v_posed, 1] + transl
 *   vertices = (o_x, -o_z, o_y) * enlargement
 * Forward: three launches; writes `vertices` and zeroes `vertices_grad` when that is not NULL.  Backward: three launches; reads
 * dL/dvertices from `vertices_grad` and WRITES (does not accumulate) the six parameter gradients.  The backward reads the
 * workspace the forward filled, so it must follow a forward with the same arguments.  Fixed-order reductions, no float
 * atomics: the same inputs give the same bits.  GMS_E_ARG before any launch: n_joints != 5, parents[0] != -1 or
 * parents[j] not in [0, j), V <= 0, n_shape outside [0, 300], n_exp outside [0, 100], a null or non-4-byte-aligned
 * pointer that the call reads or writes, or a short workspace.  Caller's stream, no host synchronisation. */
#define GMS_FLAME_JOINTS 5
typedef struct gms_flame_lbs_args {
    int32_t V, n_shape, n_exp, n_joints;
    int32_t parents[GMS_FLAME_JOINTS];  /* kintree_table[0] with parents[0] = -1 */
    const float* v_template;     /* [V,3] */
    const float* shapedirs;      /* [n_shape + n_exp, 3V]: the active columns of FLAME's [V,3,400], packed row-major */
    const float* posedirs;       /* [36, 3V] (FLAME.__init__'s layout) */
    const float* J_regressor;    /* [5, V] dense */
    const float* lbs_weights;    /* [V, 5] */
    const float* shape;          /* [n_shape] */
    const float* expression;     /* [n_exp] */
    const float* pose;           /* [6]: global rotation, jaw */
    const float* neck_pose;      /* [3] */
    const float* transl;         /* [3] */
    const float* enlargement;    /* [V,3] _vertices_enlargement */
    float* vertices;             /* [V,3] forward output */
    float* vertices_grad;        /* [V,3] forward: zeroed (may be NULL); backward: dL/dvertices */
    float* d_shape;              /* [n_shape] */
    float* d_expression;         /* [n_exp] */
    float* d_pose;               /* [6] */
    float* d_neck_pose;          /* [3] */
    float* d_transl;             /* [3] */
    float* d_enlargement;        /* [V,3] */
    void* workspace; size_t workspace_bytes;   /* gms_flame_lbs_workspace_bytes(V) */
} gms_flame_lbs_args;
size_t gms_flame_lbs_workspace_bytes(int32_t V);
int gms_flame_lbs_forward(const gms_flame_lbs_args* a, void* cuda_stream);
int gms_flame_lbs_backward(const gms_flame_lbs_args* a, void* cuda_stream);

/* Scores an image against its ground truth, forward only, deterministically (per-tile partial sums added in a fixed order in
 * double, no atomics: the same inputs give the same bits).  Both images go through the same transform first:
 *   quantize 0: clamp to [0,1]                                  (training_report, train.py:203-204)
 *   quantize 1: save_image's 8-bit rounding, back to byte / 255 (scripts/render.py's PNGs as metrics.py reads them)
 * out (device, double [4]):
 *   0  L1 = mean |x - y|                                                   (utils/loss_utils.py:17)
 *   1  SSIM, 11x11 Gaussian window sigma 1.5, zero padding, mean           (utils/loss_utils.py:33-64, metrics.py:72)
 *   2  PSNR over all channels, -10 log10(mean (x - y)^2)                   (utils/image_utils.py:17-19 on [1,C,H,W], metrics.py:73)
 *   3  mean over channels of the per-channel PSNR                          (the same psnr on a [C,H,W] tensor, train.py:212)
 * A PSNR is +inf where the MSE is 0. */
typedef struct gms_metrics_args {
    int32_t C, H, W;            /* C <= 4 */
    const float* img;           /* [C,H,W] */
    const float* gt;            /* [C,H,W] */
    int32_t quantize;           /* 0 or 1, see above */
    double* out;                /* device [4] */
    void* scratch;              /* gms_metrics_scratch_bytes() bytes */
    size_t scratch_bytes;
} gms_metrics_args;
int gms_metrics_scratch_bytes(int32_t C, int32_t H, int32_t W, size_t* bytes);
int gms_image_metrics(const gms_metrics_args* a, void* cuda_stream);

/* LPIPS of an image against its ground truth: lpips(render, gt, net_type='vgg') (lpipsPyTorch, metrics.py:74), version 0.1,
 * forward only, deterministically (per-block partial sums added in a fixed order in double, no atomics).  Both images are
 * float [3,H,W] as the reference's tensors hold them (to_tensor of the PNG: byte / 255); they are not mapped to [-1,1].
 * out (device, float [6]): the five layer terms (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3), then their sum, LPIPS.
 * Packed weights (float, GMS_LPIPS_WEIGHT_FLOATS), in this order:
 *   for each of the 13 convs of torchvision's vgg16().features (Cin -> Cout: 3->64, 64->64, 64->128, 128->128, 128->256,
 *   256->256 twice, 256->512, 512->512 five times): the weight [Cout][Kp] with K ordered (ky, kx, ci), i.e.
 *   weight.permute(0, 2, 3, 1) flattened, Kp = 9 * Cin, except conv1_1's Kp = 32 (27 values, then 5 zeros); then the bias
 *   [Cout].  Then the lin weights lin0..lin4 (vgg.pth's lin{l}.model.1.weight), 64 + 128 + 256 + 512 + 512 floats.
 * H or W < 16 (relu5_3 would be empty), a null pointer or scratch smaller than gms_lpips_scratch_bytes(H, W) is
 * GMS_E_ARG, returned without a launch.  Caller's stream, no host synchronisation. */
#define GMS_LPIPS_WEIGHT_FLOATS 14716480
typedef struct gms_lpips_args {
    int32_t H, W;               /* >= 16 */
    const float* img;           /* [3,H,W] */
    const float* gt;            /* [3,H,W] */
    const float* weights;       /* packed, see above */
    float* out;                 /* device [6] */
    void* scratch;              /* gms_lpips_scratch_bytes(H, W) bytes */
    size_t scratch_bytes;
} gms_lpips_args;
/* Scratch of gms_lpips_vgg at H x W (two [2,H,W,64] activation buffers and the partial sums); 0 when H or W < 16. */
size_t gms_lpips_scratch_bytes(int32_t H, int32_t W);
int gms_lpips_vgg(const gms_lpips_args* a, void* cuda_stream);

/* ---- image sink / source (SURVEY.md section 8(f) rank 4) ---------------------------------------- */

/* float [C,H,W] -> 8-bit interleaved rows, byte = clamp(x * 255 + 0.5, 0, 255) truncated: the device half of
 * torchvision.utils.save_image (scripts/render_time_animated.py:86-87, scripts/render.py) in one pass.  Output row stride is
 * row_prefix + W*C bytes; row_prefix = 1 reserves PNG's filter byte (written 0), 0 gives plain HWC (PPM / raw video). */
int gms_image_quantize(const float* chw, uint8_t* out, int32_t C, int32_t H, int32_t W, int32_t row_prefix, void* cuda_stream);
/* float [C,H,W] -> uint8 [H,W,C], byte = (uint8)(int64)(clamp(x, 0, 1) * 255): the bytes of the remote viewer's
 * `(torch.clamp(img, 0, 1) * 255).byte().permute(1, 2, 0).contiguous()` (train.py:72-74) on the device, bit for bit, NaN
 * and +-inf included.  It truncates where gms_image_quantize rounds.  Bad sizes (C outside 1..4, H outside 1..65535,
 * W < 1) or a null pointer are GMS_E_ARG, returned without a launch.  Caller's stream, no host synchronisation. */
int gms_image_clamp_u8(const float* chw, uint8_t* hwc, int32_t C, int32_t H, int32_t W, void* cuda_stream);
/* 8-bit image ([H,W,C] if src_is_hwc else [C,H,W]) -> float [C,H,W] = byte / 255 (ToTensor / PILtoTorch,
 * utils/general_utils.py:105-112): ground-truth images can stay 8-bit on the host and on the device. */
int gms_image_dequantize(const uint8_t* src, int32_t src_is_hwc, float* chw, int32_t C, int32_t H, int32_t W, void* cuda_stream);

/* ---- ground-truth preparation (the dataset loader, DESIGN.md 4.6) -------------------------------- */

/* uint8 RGBA [H,W,4] (4-byte aligned) -> uint8 RGB [H,W,3] over a black (white_background 0) or white (1) background,
 * bit-identical to readCamerasFromTransforms' numpy sequence (scene/dataset_readers.py:204-210): u / 255.0 in double,
 * rgb * a + bg * (1 - a), * 255.0, truncated to a byte.  Bad sizes, a null or misaligned pointer or another background
 * value are GMS_E_ARG, returned without a launch.  Caller's stream, no host synchronisation. */
int gms_image_composite_rgba(const uint8_t* rgba, uint8_t* rgb, int32_t H, int32_t W, int32_t white_background, void* cuda_stream);

/* Bicubic resample of a uint8 [in_h,in_w,3] image to [out_h,out_w,3], bit-exact to Pillow's Image.resize with its default
 * filter (PILtoTorch, utils/general_utils.py:101-107, as loadCam calls it, utils/camera_utils.py:19-52): Pillow's two-pass
 * ImagingResample, 8-bit path.  A pass runs only when its dimension changes; the horizontal pass runs first, and when both
 * run it covers only the source rows [row0, row0 + rows) the vertical pass reads, into `scratch` (out_w * rows * 3 bytes).
 * The per-axis tables come from the host (gms_b200/dataset.py resize_coeffs): bounds [out,2] = (first source index, taps),
 * coeffs [out,ksize] int32 weights in 22-bit fixed point; the kernels only do integer multiply-adds.  A table is read only
 * when its axis changes; the same size on both axes is a device copy.  Bad sizes (C != 3, a size < 1, out_h, in_h > 65535),
 * a missing table or a bad row range / short scratch are GMS_E_ARG, returned without a launch.  The tables' contents are not
 * checked.  Caller's stream, no host synchronisation. */
typedef struct gms_resize_args {
    int32_t in_w, in_h, out_w, out_h, C;
    const uint8_t* src;          /* [in_h,in_w,C] */
    uint8_t* dst;                /* [out_h,out_w,C] */
    const int32_t* bounds_h;     /* [out_w,2] */
    const int32_t* coeffs_h;     /* [out_w,ksize_h] */
    int32_t ksize_h;
    const int32_t* bounds_v;     /* [out_h,2], source rows of the original image */
    const int32_t* coeffs_v;     /* [out_h,ksize_v] */
    int32_t ksize_v;
    int32_t row0, rows;          /* both passes: bounds_v[0] and bounds_v[last] + taps - bounds_v[0] */
    uint8_t* scratch;
    size_t scratch_bytes;
} gms_resize_args;
int gms_image_resize_u8(const gms_resize_args* a, void* cuda_stream);

/* ---- anomaly detection (train.py --detect_anomaly) ------------------------------------------------ */

/* torch.autograd.set_detect_anomaly(True) for the one-call frames, which run without an autograd graph: the outputs of a
 * backward stage are scanned for NaN (only NaN, as torch's check: +-inf, denormals and -0 are not reported) and the first
 * one is recorded in ONE device word
 *   key = stage << 56 | tensor << 48 | element index (row-major, < 2^48),
 * the smallest key over every scan since the caller last set the word to GMS_ANOMALY_NONE: the earliest stage, then the
 * lowest tensor id, then the lowest index.  The scan reads each buffer once with 128-bit loads (scalar head and tail for any
 * 4-byte-aligned pointer and any length) and makes at most one atomicMin per thread block, only when that block saw a NaN. */
#define GMS_ANOMALY_NONE 0xFFFFFFFFFFFFFFFFull
/* stages, in the order a frame runs them */
#define GMS_ANOMALY_LOSS 0              /* the L1 + SSIM loss kernels */
#define GMS_ANOMALY_COMPOSITE_BWD 1     /* the composite backward */
#define GMS_ANOMALY_PREPROCESS_BWD 2    /* the preprocess backward */
#define GMS_ANOMALY_EXPAND_BWD 3        /* the mesh expansion backward (gms_train_frame), after every segment */
#define GMS_ANOMALY_ACTIVATION_BWD 4    /* the scale / rotation activation backward (gms_free_train_frame) */
#define GMS_ANOMALY_FLAME_BWD 5         /* gms_flame_lbs_backward (scanned by the caller through gms_nan_scan) */
#define GMS_ANOMALY_STAGES 6
/* tensors of each stage */
#define GMS_ANOMALY_DIMAGE 0            /* LOSS: dL/dimage [3,H,W] */
#define GMS_ANOMALY_DGEOM 0             /* COMPOSITE_BWD: the per-Gaussian gradient records [P,12] (gms_debug_views.dgeom) */
#define GMS_ANOMALY_DMEANS3D 0          /* PREPROCESS_BWD: [P,3] */
#define GMS_ANOMALY_DSCALES 1           /*   [P,3] w.r.t. the activated scales */
#define GMS_ANOMALY_DROTATIONS 2        /*   [P,4] w.r.t. the unit quaternions */
#define GMS_ANOMALY_DOPACITY_RAW 3      /*   [P,1] w.r.t. the opacity logits */
#define GMS_ANOMALY_DSHS 4              /*   [P,M,3] SH gradient rows (d_features) */
#define GMS_ANOMALY_DCOLOR_SH 5         /*   [P,3] factored colour gradient (d_color_sh) */
#define GMS_ANOMALY_DVERTICES 0         /* EXPAND_BWD: [V,3] (accumulated: includes whatever the caller left in it) */
#define GMS_ANOMALY_DALPHA_RAW 1        /*   [P,3] */
#define GMS_ANOMALY_DSCALE_RAW 2        /*   [P,1] */
#define GMS_ANOMALY_DSCALING_RAW 0      /* ACTIVATION_BWD: [P,scale_cols] */
#define GMS_ANOMALY_DROTATION_RAW 1     /*   [P,4] */
#define GMS_ANOMALY_ACCUM 2             /*   [P] densification statistic (when gathered) */
#define GMS_ANOMALY_DSHAPE 0            /* FLAME_BWD: [n_shape] */
#define GMS_ANOMALY_DEXPRESSION 1       /*   [n_exp] */
#define GMS_ANOMALY_DPOSE 2             /*   [6] */
#define GMS_ANOMALY_DNECK_POSE 3        /*   [3] */
#define GMS_ANOMALY_DTRANSL 4           /*   [3] */
#define GMS_ANOMALY_DENLARGEMENT 5      /*   [V,3] */
#define GMS_NAN_SCAN_MAX_BUFFERS 8
typedef struct gms_nan_buffer {
    const float* ptr;           /* device, 4-byte aligned; may be NULL when n == 0 */
    int64_t n;                  /* floats, 0 <= n < 2^48 */
    int32_t tensor;             /* 0..255 */
} gms_nan_buffer;
typedef struct gms_nan_scan_args {
    gms_nan_buffer buffers[GMS_NAN_SCAN_MAX_BUFFERS];
    int32_t n_buffers;          /* 0..GMS_NAN_SCAN_MAX_BUFFERS */
    int32_t stage;              /* 0..GMS_ANOMALY_STAGES-1 */
    uint64_t* record;           /* device word; left untouched when no buffer holds a NaN */
} gms_nan_scan_args;
/* One launch over every buffer of the table (none when they are all empty).  GMS_E_ARG before any launch: a null record,
 * n < 0 or n >= 2^48, more than GMS_NAN_SCAN_MAX_BUFFERS buffers, a null or misaligned pointer with n > 0, a stage or a tensor
 * id out of range.  Caller's stream, no host synchronisation. */
int gms_nan_scan(const gms_nan_scan_args* a, void* cuda_stream);

/* ---- misc ------------------------------------------------------------------------------------- */
const char* gms_last_error(void);
const char* gms_version(void);
/* Number of kernel launches issued by this library since the last call with reset != 0 (bench.py's
 * "gpu_launches" claim is counted, not guessed). */
int64_t gms_launch_count(int reset);
/* Per-kernel device time, measured with CUDA events recorded on the launching stream around every launch made
 * while option "time_kernels" is 1.  Fills up to max_kernels entries (accumulated ms, launch count, name) and
 * returns the number of kernel slots. */
int gms_kernel_times(int reset, int max_kernels, double* ms_out, int64_t* count_out, const char** names_out);
/* Tuning knobs (round-over-round experiments): "warp_emit", "time_kernels", "composite_fwd", "composite_bwd",
 * "bwd_minblocks", "key16", "adam_sh_ieee", "tile_order", "sort_impl", "bin_impl", "sh_staged", "pre_bwd_minblocks"
 * (DESIGN.md lists what each selects).  Returns the previous value; unknown keys return -1. */
int gms_set_option(const char* key, int value);

#ifdef __cplusplus
}
#endif
#endif /* GMS_B200_H */
