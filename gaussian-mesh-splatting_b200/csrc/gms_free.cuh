// gms_free.cuh -- free Gaussians (gs, gs_flat): the per-Gaussian activation of the training frame and densification.
//
// Activation (scene/gaussian_model.py:95-101, games/flat_splatting/scene/flat_gaussian_model.py:32-35):
//   gs      get_scaling = exp(_scaling)                    [P,3]
//   gs_flat get_scaling = (eps_s0, exp(_scaling[:, -2:]))  [P,2] raw -> [P,3]
//   get_rotation = F.normalize(_rotation) = r / max(|r|, 1e-12)
// Densification (scene/gaussian_model.py:360-414, flat_gaussian_model.py:62-88) is planned per source row: one row gives at
// most one kept original, one clone, and a pair of split children (copy 0 and copy 1), each of which the final prune may
// drop.  A clone has its original's raw values, so it survives the prune exactly when the original would; both split
// children share their scaling and opacity, so they survive together.
#pragma once
#include "gms_common.cuh"

#define GMS_FREE_BLOCK 128

// dL/dscales and dL/drotations of the rasterizer -> raw-parameter gradients, plus the densification statistics of
// add_densification_stats (scene/gaussian_model.py:416-418): accum += |dL/dmean2D.xy| and denom += 1 where radii > 0.
struct FreeActBwd {
    int P, cols;
    const float* rotation_raw; const float* scales;     // scales: the activated [P,3] the forward wrote
    const float* d_scales; const float* d_rots; const float* d_m2d; const int32_t* radii;
    float* d_scaling_raw; float* d_rotation_raw;
    float* accum; float* denom;                         // NULL: no statistics
    const uint32_t* counters;                           // device [2] (N, overflow flag) of this frame's binning; NULL: none
};

__device__ __forceinline__ float gms_quat_norm(const float q[4]) {
    return fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
}

__global__ void __launch_bounds__(GMS_FREE_BLOCK) k_free_act_fwd(int P, int cols, const float* __restrict__ scaling_raw,
                                                                  const float* __restrict__ rotation_raw, float eps,
                                                                  float* __restrict__ scales, float* __restrict__ rots) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float* s = scaling_raw + (size_t)cols * i;
    float* so = scales + 3 * (size_t)i;
    if (cols == 3) { so[0] = expf(s[0]); so[1] = expf(s[1]); so[2] = expf(s[2]); }
    else { so[0] = eps; so[1] = expf(s[0]); so[2] = expf(s[1]); }
    const float4 r = reinterpret_cast<const float4*>(rotation_raw)[i];
    const float q[4] = {r.x, r.y, r.z, r.w};
    const float n = gms_quat_norm(q);
    reinterpret_cast<float4*>(rots)[i] = make_float4(q[0] / n, q[1] / n, q[2] / n, q[3] / n);
}

// xyz from the checkpoint's activated weights and the driving pose (the product of the expansion forward, same operation
// order), scales and rotations from the checkpoint's rows as k_free_act_fwd activates them.  C linkage: its symbol, and
// the name profiler traces give it, is the plain `k_flame_act`.
extern "C" __global__ void __launch_bounds__(GMS_FREE_BLOCK) k_flame_act(int P, int K, const float* __restrict__ alpha, const int64_t* __restrict__ faces,
                                                              const float* __restrict__ vertices, const float* __restrict__ scaling_log,
                                                              const float* __restrict__ rotation_raw, float* __restrict__ xyz,
                                                              float* __restrict__ scales, float* __restrict__ rots) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const size_t f = (size_t)(i / K);
    float t[9];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const int64_t vi = faces[3 * f + c];
        t[3 * c] = vertices[3 * vi]; t[3 * c + 1] = vertices[3 * vi + 1]; t[3 * c + 2] = vertices[3 * vi + 2];
    }
    const float al0 = alpha[3 * (size_t)i], al1 = alpha[3 * (size_t)i + 1], al2 = alpha[3 * (size_t)i + 2];
#pragma unroll
    for (int c = 0; c < 3; c++) xyz[3 * (size_t)i + c] = al0 * t[c] + al1 * t[3 + c] + al2 * t[6 + c];
    const float* s = scaling_log + 3 * (size_t)i;
    float* so = scales + 3 * (size_t)i;
    so[0] = expf(s[0]); so[1] = expf(s[1]); so[2] = expf(s[2]);
    const float4 r = reinterpret_cast<const float4*>(rotation_raw)[i];
    const float q[4] = {r.x, r.y, r.z, r.w};
    const float n = gms_quat_norm(q);
    reinterpret_cast<float4*>(rots)[i] = make_float4(q[0] / n, q[1] / n, q[2] / n, q[3] / n);
}

__global__ void __launch_bounds__(GMS_FREE_BLOCK) k_free_act_bwd(FreeActBwd b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b.P) return;
    // scales: d exp(x)/dx = exp(x); the eps column of gs_flat is a constant
    const float* ds = b.d_scales + 3 * (size_t)i;
    const float* sa = b.scales + 3 * (size_t)i;
    float* dsr = b.d_scaling_raw + (size_t)b.cols * i;
    if (b.cols == 3) { dsr[0] = ds[0] * sa[0]; dsr[1] = ds[1] * sa[1]; dsr[2] = ds[2] * sa[2]; }
    else { dsr[0] = ds[1] * sa[1]; dsr[1] = ds[2] * sa[2]; }
    // rotation: d(r / n)/dr = (I - u u^T) / n above the clamp, I / n below it (n = 1e-12 is then a constant)
    const float4 r = reinterpret_cast<const float4*>(b.rotation_raw)[i];
    const float4 d = reinterpret_cast<const float4*>(b.d_rots)[i];
    const float q[4] = {r.x, r.y, r.z, r.w};
    const float dq[4] = {d.x, d.y, d.z, d.w};
    const float qn = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float n = fmaxf(qn, 1e-12f);
    float o[4];
    if (qn >= 1e-12f) {
        const float u[4] = {q[0] / n, q[1] / n, q[2] / n, q[3] / n};
        const float dd = dq[0] * u[0] + dq[1] * u[1] + dq[2] * u[2] + dq[3] * u[3];
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = (dq[k] - u[k] * dd) / n;
    } else {
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = dq[k] / n;
    }
    reinterpret_cast<float4*>(b.d_rotation_raw)[i] = make_float4(o[0], o[1], o[2], o[3]);
    // statistics: nothing on an overflowed frame (its image is the background and its gradients are zero)
    if (b.accum && b.radii[i] > 0 && !(b.counters && b.counters[1])) {
        const float gx = b.d_m2d[3 * (size_t)i], gy = b.d_m2d[3 * (size_t)i + 1];
        b.accum[i] += sqrtf(gx * gx + gy * gy);
        b.denom[i] += 1.f;
    }
}

// ---- densification

struct DensifyPlanK {
    int P, cols;
    const float* accum; const float* denom; const float* scaling_raw; const float* opacity_raw;
    float eps, grad_threshold, split_scale, min_opacity, max_world_scale;   // max_world_scale <= 0: no size prune
    int4* flags;            // out [P]: (kept original, surviving clone, surviving split pair, pruned rows)
    uint8_t* fate;          // out [P] or NULL: GMS_FATE_* bits
};

// IEEE single-precision arithmetic without contraction, as ATen's CPU kernels evaluate these expressions
__device__ __forceinline__ float gms_sigmoid(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

__device__ __forceinline__ float free_max_scale(const float* s, int cols, float eps) {
    return cols == 3 ? fmaxf(fmaxf(expf(s[0]), expf(s[1])), expf(s[2])) : fmaxf(fmaxf(eps, expf(s[0])), expf(s[1]));
}

// log(get_scaling / (0.8 * N)) of a split child, N = 2 (for gs_flat the columns [1, 2] of it)
__device__ __forceinline__ float free_child_log_scale(float raw) { return logf(__fdiv_rn(expf(raw), 1.6f)); }

__global__ void __launch_bounds__(GMS_FREE_BLOCK) k_densify_plan(DensifyPlanK a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    float g = __fdiv_rn(a.accum[i], a.denom[i]);
    if (isnan(g)) g = 0.f;
    const float* s = a.scaling_raw + (size_t)a.cols * i;
    const float smax = free_max_scale(s, a.cols, a.eps);
    const bool hot = g >= a.grad_threshold;
    const bool clone = hot && smax <= a.split_scale, split = hot && smax > a.split_scale;
    const bool transparent = gms_sigmoid(a.opacity_raw[i]) < a.min_opacity;
    const bool size_prune = a.max_world_scale > 0.f;
    const bool prune = transparent || (size_prune && smax > a.max_world_scale);
    bool prune_child = transparent;
    if (split && size_prune) {
        float c[3];
        for (int k = 0; k < a.cols; k++) c[k] = free_child_log_scale(s[k]);
        prune_child = prune_child || free_max_scale(c, a.cols, a.eps) > a.max_world_scale;
    }
    int4 f;
    f.x = !split && !prune;
    f.y = clone && !prune;
    f.z = split && !prune_child;
    f.w = (!split && prune) + (clone && prune) + 2 * (split && prune_child);
    a.flags[i] = f;
    if (a.fate) a.fate[i] = (uint8_t)((clone ? 1 : 0) | (split ? 2 : 0) | (prune ? 4 : 0) | (split && prune_child ? 8 : 0));
}

struct Int4Sum {
    __device__ __forceinline__ int4 operator()(const int4& a, const int4& b) const {
        return make_int4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    }
};

struct FreeSetK { const float* xyz; const float* scaling; const float* rotation; const float* opacity; const float* features; };
struct FreeSetOutK { float* xyz; float* scaling; float* rotation; float* opacity; float* features; };

struct DensifyApplyK {
    int P, cols, F;            // F = 3 * M floats of features per row
    float eps;
    const int4* incl;          // inclusive scan of the plan's flags
    int kept, clones, splits;  // totals: output rows [0, kept) originals, then clones, then copy 0, then copy 1
    const float* normals;      // [P,2,3]
    FreeSetK src[3];
    FreeSetOutK dst[3];
};

// One destination row: parameters copied from source row i (moments too when `moments`; zero otherwise).
__device__ __forceinline__ void densify_copy_row(const DensifyApplyK& a, int i, int o, bool moments) {
    for (int t = 0; t < 3; t++) {
        const FreeSetK& s = a.src[t];
        const FreeSetOutK& d = a.dst[t];
        const bool z = t > 0 && !moments;
        for (int k = 0; k < 3; k++) d.xyz[3 * (size_t)o + k] = z ? 0.f : s.xyz[3 * (size_t)i + k];
        for (int k = 0; k < a.cols; k++) d.scaling[(size_t)a.cols * o + k] = z ? 0.f : s.scaling[(size_t)a.cols * i + k];
        for (int k = 0; k < 4; k++) d.rotation[4 * (size_t)o + k] = z ? 0.f : s.rotation[4 * (size_t)i + k];
        d.opacity[o] = z ? 0.f : s.opacity[i];
        for (int k = 0; k < a.F; k++) d.features[(size_t)a.F * o + k] = z ? 0.f : s.features[(size_t)a.F * i + k];
    }
}

__global__ void __launch_bounds__(GMS_FREE_BLOCK) k_densify_apply(DensifyApplyK a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    const int4 hi = a.incl[i];
    const int4 lo = i > 0 ? a.incl[i - 1] : make_int4(0, 0, 0, 0);
    if (hi.x != lo.x) densify_copy_row(a, i, lo.x, true);
    if (hi.y != lo.y) densify_copy_row(a, i, a.kept + lo.y, false);
    if (hi.z == lo.z) return;
    // split children: xyz = R(q) (std * z) + xyz with std = get_scaling, scaling = log(get_scaling / 1.6)
    const float* sr = a.src[0].scaling + (size_t)a.cols * i;
    const float std[3] = {a.cols == 3 ? expf(sr[0]) : a.eps, expf(sr[a.cols - 2]), expf(sr[a.cols - 1])};
    const float* r = a.src[0].rotation + 4 * (size_t)i;
    // build_rotation (utils/general_utils.py:158-179), one rounding per operation as ATen evaluates it
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], r[0]), __fmul_rn(r[1], r[1])), __fmul_rn(r[2], r[2])),
                                           __fmul_rn(r[3], r[3])));
    const float w = __fdiv_rn(r[0], nrm), x = __fdiv_rn(r[1], nrm), y = __fdiv_rn(r[2], nrm), z = __fdiv_rn(r[3], nrm);
    const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
    const float wx = __fmul_rn(w, x), wy = __fmul_rn(w, y), wz = __fmul_rn(w, z);
    const float R[9] = {__fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(yy, zz))), __fmul_rn(2.f, __fsub_rn(xy, wz)), __fmul_rn(2.f, __fadd_rn(xz, wy)),
                        __fmul_rn(2.f, __fadd_rn(xy, wz)), __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, zz))), __fmul_rn(2.f, __fsub_rn(yz, wx)),
                        __fmul_rn(2.f, __fsub_rn(xz, wy)), __fmul_rn(2.f, __fadd_rn(yz, wx)), __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, yy)))};
    float child_s[3];
#pragma unroll
    for (int k = 0; k < 3; k++) child_s[k] = k < a.cols ? free_child_log_scale(sr[k]) : 0.f;
    const float* xyz = a.src[0].xyz + 3 * (size_t)i;
    for (int c = 0; c < 2; c++) {
        const int o = a.kept + a.clones + c * a.splits + lo.z;
        densify_copy_row(a, i, o, false);
        const float* zn = a.normals + 6 * (size_t)i + 3 * c;
        const float smp[3] = {__fmul_rn(zn[0], std[0]), __fmul_rn(zn[1], std[1]), __fmul_rn(zn[2], std[2])};
        for (int k = 0; k < 3; k++)
            a.dst[0].xyz[3 * (size_t)o + k] =
                __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[3 * k], smp[0]), __fmul_rn(R[3 * k + 1], smp[1])), __fmul_rn(R[3 * k + 2], smp[2])), xyz[k]);
#pragma unroll
        for (int k = 0; k < 3; k++)
            if (k < a.cols) a.dst[0].scaling[(size_t)a.cols * o + k] = child_s[k];
    }
}
