// gms_flame.cuh -- FLAME's vertex model (linear blend skinning) forward and backward, sm_90a.
//
// The computation is FLAME.forward (games/flame_splatting/FLAME/FLAME.py:204-248, smplx.lbs.lbs) followed by
// transform_vertices_function (games/flame_splatting/scene/dataset_readers.py:40-45), for one frame:
//   v_shaped = v_template + shapedirs . betas          (only the n_shape + n_exp active columns, packed [B,3V])
//   J        = J_regressor [5,V] . v_shaped
//   R_j      = rodrigues(full_pose_j), full_pose = [pose[:3], neck, pose[3:], eyes = 0]
//   v_posed  = v_shaped + ((R_1..4 - I) flattened, 36 values) . posedirs [36,3V]
//   G_j      = G_parent(j) . [R_j | J_j - J_parent(j)],  A_j = G_j with the rest joint removed (t -= G_j,r J_j)
//   o        = (sum_j w_vj A_j) . [v_posed, 1] + transl
//   out      = (o_x, -o_z, o_y) * enlargement[v]
// The joint part (Rodrigues, the chain and their backward) is a handful of 3x3 products for five joints: one thread does it,
// and the device functions below compile for the host too (tests/hostshim checks them against float64).  Every reduction
// over vertices runs in a fixed order (warp butterflies, then per-warp or per-block partials summed sequentially): no float
// atomics, so the same inputs give the same bits.
#pragma once
#include "gms_common.cuh"

#define GMS_FLAME_NJ 5            // joints: global, neck, jaw, left eye, right eye
#define GMS_FLAME_NFEAT 36        // pose features: (R_j - I) of joints 1..4
#define GMS_FLAME_RED 99          // per-block backward partials: dtransl (3), dA (5 x 12), dfeat (36)

// Everything the joint stage produces, one per frame.
struct GmsFlameJoints {
    float R[GMS_FLAME_NJ][9];     // rotation per joint, row-major
    float G[GMS_FLAME_NJ][12];    // world transform per joint, rows 0..2 of the 4x4 (row 3 is 0 0 0 1)
    float A[GMS_FLAME_NJ][12];    // G with the rest joint removed: A[:, 3] = G[:, 3] - G[:, :3] J_j
    float feat[GMS_FLAME_NFEAT];  // (R_j - I) flattened, j = 1..4
};

// smplx.lbs.batch_rodrigues for one axis-angle: angle = |rv + 1e-8|, k = rv / angle, R = I + sin K + (1 - cos) K K.
GMS_HD void gms_flame_rodrigues(const float rv[3], float R[9]) {
    const float a0 = rv[0] + 1e-8f, a1 = rv[1] + 1e-8f, a2 = rv[2] + 1e-8f;
    const float angle = sqrtf(a0 * a0 + a1 * a1 + a2 * a2);
    const float kx = rv[0] / angle, ky = rv[1] / angle, kz = rv[2] / angle;
    const float s = sinf(angle), omc = 1.0f - cosf(angle);
    const float K[9] = {0.f, -kz, ky, kz, 0.f, -kx, -ky, kx, 0.f};
    for (int r = 0; r < 3; r++)
        for (int q = 0; q < 3; q++) {
            const float kk = K[3 * r] * K[q] + K[3 * r + 1] * K[3 + q] + K[3 * r + 2] * K[6 + q];
            R[3 * r + q] = (r == q ? 1.0f : 0.0f) + s * K[3 * r + q] + omc * kk;
        }
}

// d(rv) of gms_flame_rodrigues for an upstream dR, by the chain rule through the same operations.
GMS_HD void gms_flame_rodrigues_bwd(const float rv[3], const float dR[9], float drv[3]) {
    const float a0 = rv[0] + 1e-8f, a1 = rv[1] + 1e-8f, a2 = rv[2] + 1e-8f;
    const float angle = sqrtf(a0 * a0 + a1 * a1 + a2 * a2);
    const float kx = rv[0] / angle, ky = rv[1] / angle, kz = rv[2] / angle;
    const float s = sinf(angle), c = cosf(angle), omc = 1.0f - c;
    const float K[9] = {0.f, -kz, ky, kz, 0.f, -kx, -ky, kx, 0.f};
    float ds = 0.f, domc = 0.f, dK[9];
    for (int r = 0; r < 3; r++)
        for (int q = 0; q < 3; q++) {
            const float kk = K[3 * r] * K[q] + K[3 * r + 1] * K[3 + q] + K[3 * r + 2] * K[6 + q];
            ds += dR[3 * r + q] * K[3 * r + q];
            domc += dR[3 * r + q] * kk;
        }
    // d(K K) = dR (1 - cos): dK = sin dR + (1 - cos) (dR K^T + K^T dR)
    for (int r = 0; r < 3; r++)
        for (int q = 0; q < 3; q++) {
            float m = 0.f;
            for (int t = 0; t < 3; t++) m += dR[3 * r + t] * K[3 * q + t] + K[3 * t + r] * dR[3 * t + q];
            dK[3 * r + q] = s * dR[3 * r + q] + omc * m;
        }
    const float dkx = dK[7] - dK[5], dky = dK[2] - dK[6], dkz = dK[3] - dK[1];
    // s = sin(angle), omc = 1 - cos(angle), k = rv / angle
    float dangle = ds * c + domc * s;
    dangle -= (dkx * rv[0] + dky * rv[1] + dkz * rv[2]) / (angle * angle);
    const float g = dangle / angle;     // angle = |a|: d a = dangle a / angle
    drv[0] = dkx / angle + g * a0;
    drv[1] = dky / angle + g * a1;
    drv[2] = dkz / angle + g * a2;
}

// The full pose of joint j from the frame's parameters (eyes fixed at zero, as FLAME's default eye_pose).
GMS_HD void gms_flame_joint_rv(int j, const float pose[6], const float neck[3], float rv[3]) {
    for (int c = 0; c < 3; c++)
        rv[c] = j == 0 ? pose[c] : j == 1 ? neck[c] : j == 2 ? pose[3 + c] : 0.0f;
}

// Rodrigues, the chain (smplx.lbs.batch_rigid_transform) and the pose feature for the joint positions J [5][3].
GMS_HD void gms_flame_joints_fwd(const float pose[6], const float neck[3], const float J[15], const int32_t parents[GMS_FLAME_NJ],
                                 GmsFlameJoints& o) {
    for (int j = 0; j < GMS_FLAME_NJ; j++) {
        float rv[3];
        gms_flame_joint_rv(j, pose, neck, rv);
        gms_flame_rodrigues(rv, o.R[j]);
    }
    for (int j = 0; j < GMS_FLAME_NJ; j++) {
        const int p = parents[j];
        const float* R = o.R[j];
        float rel[3];
        for (int c = 0; c < 3; c++) rel[c] = p < 0 ? J[3 * j + c] : J[3 * j + c] - J[3 * p + c];
        float* G = o.G[j];
        if (p < 0) {
            for (int r = 0; r < 3; r++) {
                for (int q = 0; q < 3; q++) G[4 * r + q] = R[3 * r + q];
                G[4 * r + 3] = rel[r];
            }
        } else {
            const float* P = o.G[p];
            for (int r = 0; r < 3; r++) {
                for (int q = 0; q < 3; q++) G[4 * r + q] = P[4 * r] * R[q] + P[4 * r + 1] * R[3 + q] + P[4 * r + 2] * R[6 + q];
                G[4 * r + 3] = P[4 * r] * rel[0] + P[4 * r + 1] * rel[1] + P[4 * r + 2] * rel[2] + P[4 * r + 3];
            }
        }
        for (int r = 0; r < 3; r++) {
            for (int q = 0; q < 3; q++) o.A[j][4 * r + q] = G[4 * r + q];
            o.A[j][4 * r + 3] = G[4 * r + 3] - (G[4 * r] * J[3 * j] + G[4 * r + 1] * J[3 * j + 1] + G[4 * r + 2] * J[3 * j + 2]);
        }
    }
    for (int j = 1; j < GMS_FLAME_NJ; j++)
        for (int e = 0; e < 9; e++) o.feat[9 * (j - 1) + e] = o.R[j][e] - ((e % 4) == 0 ? 1.0f : 0.0f);
}

// Backward of gms_flame_joints_fwd: dA [5][12] and dfeat [36] -> d pose [6], d neck [3], dJ [15].  `o` is the forward's.
GMS_HD void gms_flame_joints_bwd(const float pose[6], const float neck[3], const float J[15], const int32_t parents[GMS_FLAME_NJ],
                                 const GmsFlameJoints& o, const float dA[GMS_FLAME_NJ * 12], const float dfeat[GMS_FLAME_NFEAT],
                                 float dpose[6], float dneck[3], float dJ[15]) {
    float dG[GMS_FLAME_NJ][12], dR[GMS_FLAME_NJ][9];
    for (int k = 0; k < 15; k++) dJ[k] = 0.f;
    // A = [G_r | G_t - G_r J]
    for (int j = 0; j < GMS_FLAME_NJ; j++) {
        const float* d = dA + 12 * j;
        const float* G = o.G[j];
        for (int r = 0; r < 3; r++) {
            for (int q = 0; q < 3; q++) dG[j][4 * r + q] = d[4 * r + q] - d[4 * r + 3] * J[3 * j + q];
            dG[j][4 * r + 3] = d[4 * r + 3];
        }
        for (int q = 0; q < 3; q++) dJ[3 * j + q] -= G[q] * d[3] + G[4 + q] * d[7] + G[8 + q] * d[11];
    }
    // the chain, leaves first (parents[j] < j)
    for (int j = GMS_FLAME_NJ - 1; j >= 0; j--) {
        const int p = parents[j];
        float drel[3];
        if (p < 0) {
            for (int r = 0; r < 3; r++) {
                for (int q = 0; q < 3; q++) dR[j][3 * r + q] = dG[j][4 * r + q];
                drel[r] = dG[j][4 * r + 3];
            }
        } else {
            const float* P = o.G[p];
            const float* R = o.R[j];
            float rel[3];
            for (int c = 0; c < 3; c++) rel[c] = J[3 * j + c] - J[3 * p + c];
            for (int m = 0; m < 3; m++) {
                for (int q = 0; q < 3; q++) dR[j][3 * m + q] = P[m] * dG[j][q] + P[4 + m] * dG[j][4 + q] + P[8 + m] * dG[j][8 + q];
                drel[m] = P[m] * dG[j][3] + P[4 + m] * dG[j][7] + P[8 + m] * dG[j][11];
            }
            for (int r = 0; r < 3; r++) {
                for (int m = 0; m < 3; m++)
                    dG[p][4 * r + m] += dG[j][4 * r] * R[3 * m] + dG[j][4 * r + 1] * R[3 * m + 1] + dG[j][4 * r + 2] * R[3 * m + 2] +
                                        dG[j][4 * r + 3] * rel[m];
                dG[p][4 * r + 3] += dG[j][4 * r + 3];
            }
        }
        for (int c = 0; c < 3; c++) {
            dJ[3 * j + c] += drel[c];
            if (p >= 0) dJ[3 * p + c] -= drel[c];
        }
    }
    for (int j = 1; j < GMS_FLAME_NJ; j++)
        for (int e = 0; e < 9; e++) dR[j][e] += dfeat[9 * (j - 1) + e];
    for (int j = 0; j < 3; j++) {           // the eyes' gradients are discarded (their pose is fixed)
        float rv[3], drv[3];
        gms_flame_joint_rv(j, pose, neck, rv);
        gms_flame_rodrigues_bwd(rv, dR[j], drv);
        for (int c = 0; c < 3; c++) {
            if (j == 0) dpose[c] = drv[c];
            else if (j == 1) dneck[c] = drv[c];
            else dpose[3 + c] = drv[c];
        }
    }
}

#if defined(__CUDACC__)

#define GMS_FLAME_VB 128          // vertices per block of the per-vertex passes
#define GMS_FLAME_SB 64           // vertices per block of the shape pass (3 threads per vertex)

// Workspace, in floats, 64-float aligned sections (gms_flame_lbs_workspace_bytes).
struct GmsFlameWs {
    float* vs;        // [3V] v_shaped
    float* vp;        // [3V] v_posed
    float* dvp;       // [3V] dL/dv_posed
    float* jpart;     // [nsb][15] block partials of J
    float* J;         // [16]
    float* state;     // GmsFlameJoints
    float* bpart;     // [nvb][GMS_FLAME_RED] block partials of the backward
    float* dJ;        // [16]
    size_t floats;
};

static inline size_t gms_flame_pad(size_t n) { return (n + 63) / 64 * 64; }

static inline GmsFlameWs gms_flame_ws(float* base, int V) {
    const size_t nsb = (size_t)(V + GMS_FLAME_SB - 1) / GMS_FLAME_SB, nvb = (size_t)(V + GMS_FLAME_VB - 1) / GMS_FLAME_VB;
    GmsFlameWs w;
    size_t off = 0;
    auto take = [&](size_t n) { float* p = base ? base + off : nullptr; off += gms_flame_pad(n); return p; };
    w.vs = take(3 * (size_t)V); w.vp = take(3 * (size_t)V); w.dvp = take(3 * (size_t)V);
    w.jpart = take(15 * nsb); w.J = take(16);
    w.state = take((sizeof(GmsFlameJoints) + 3) / 4);
    w.bpart = take(GMS_FLAME_RED * nvb); w.dJ = take(16);
    w.floats = off;
    return w;
}

// Butterfly sum over a warp: every lane ends with the same value, added in the same order on every call.
__device__ __forceinline__ float gms_flame_warp_sum(float x) {
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// Forward 1: v_shaped, one thread per coordinate (the [B,3V] basis rows read coalesced), and per-block partials of J.
__global__ void __launch_bounds__(3 * GMS_FLAME_SB) k_flame_shape(int V, int n_shape, int n_exp, const float* __restrict__ v_template,
                                                                 const float* __restrict__ shapedirs, const float* __restrict__ shape,
                                                                 const float* __restrict__ expr, const float* __restrict__ Jreg,
                                                                 float* __restrict__ vs, float* __restrict__ jpart) {
    __shared__ float betas[400];
    __shared__ float prod[GMS_FLAME_NJ][3 * GMS_FLAME_SB];
    const int B = n_shape + n_exp;
    for (int b = threadIdx.x; b < B; b += blockDim.x) betas[b] = b < n_shape ? shape[b] : expr[b - n_shape];
    __syncthreads();
    const size_t n3 = 3 * (size_t)V;
    const size_t i = (size_t)blockIdx.x * 3 * GMS_FLAME_SB + threadIdx.x;
    float x = 0.f;
    if (i < n3) {
        float acc = 0.f;
#pragma unroll 4
        for (int b = 0; b < B; b++) acc = fmaf(betas[b], __ldg(shapedirs + (size_t)b * n3 + i), acc);
        x = v_template[i] + acc;
        vs[i] = x;
    }
    const int v = (int)(i / 3);
#pragma unroll
    for (int j = 0; j < GMS_FLAME_NJ; j++) prod[j][threadIdx.x] = i < n3 ? Jreg[(size_t)j * V + v] * x : 0.f;
    __syncthreads();
    if (threadIdx.x < 15) {
        const int j = threadIdx.x / 3, c = threadIdx.x % 3;
        float s = 0.f;
        for (int u = 0; u < GMS_FLAME_SB; u++) s += prod[j][3 * u + c];
        jpart[(size_t)blockIdx.x * 15 + threadIdx.x] = s;
    }
}

struct GmsFlameParents { int32_t p[GMS_FLAME_NJ]; };

// Forward 2 (one block): J in block order, then the joint stage.
__global__ void k_flame_joints(int nsb, const float* __restrict__ jpart, const float* __restrict__ pose,
                               const float* __restrict__ neck, GmsFlameParents par, float* __restrict__ J, float* __restrict__ state) {
    __shared__ float sJ[15];
    if (threadIdx.x < 15) {
        float s = 0.f;
        for (int b = 0; b < nsb; b++) s += jpart[(size_t)b * 15 + threadIdx.x];
        sJ[threadIdx.x] = s;
        J[threadIdx.x] = s;
    }
    __syncthreads();
    __shared__ GmsFlameJoints o;
    if (threadIdx.x == 0) {
        float p[6], n[3];
        for (int k = 0; k < 6; k++) p[k] = pose[k];
        for (int k = 0; k < 3; k++) n[k] = neck[k];
        gms_flame_joints_fwd(p, n, sJ, par.p, o);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < (int)(sizeof(GmsFlameJoints) / 4); k += blockDim.x) state[k] = reinterpret_cast<const float*>(&o)[k];
}

// Forward 3: pose offsets, skinning, transl, the axis swap and the enlargement; zeroes the frame's vertex gradient.
__global__ void __launch_bounds__(GMS_FLAME_VB) k_flame_skin(int V, const float* __restrict__ vs, const float* __restrict__ posedirs,
                                                            const float* __restrict__ weights, const float* __restrict__ transl,
                                                            const float* __restrict__ enl, const float* __restrict__ state,
                                                            float* __restrict__ vp_out, float* __restrict__ out, float* __restrict__ vgrad) {
    __shared__ float A[GMS_FLAME_NJ * 12], feat[GMS_FLAME_NFEAT], t[3];
    const GmsFlameJoints* st = reinterpret_cast<const GmsFlameJoints*>(state);
    for (int k = threadIdx.x; k < GMS_FLAME_NJ * 12; k += blockDim.x) A[k] = (&st->A[0][0])[k];
    for (int k = threadIdx.x; k < GMS_FLAME_NFEAT; k += blockDim.x) feat[k] = st->feat[k];
    if (threadIdx.x < 3) t[threadIdx.x] = transl[threadIdx.x];
    __syncthreads();
    const int v = blockIdx.x * GMS_FLAME_VB + threadIdx.x;
    if (v >= V) return;
    const size_t n3 = 3 * (size_t)V;
    float p[3];
    for (int c = 0; c < 3; c++) {
        float acc = 0.f;
#pragma unroll 4
        for (int k = 0; k < GMS_FLAME_NFEAT; k++) acc = fmaf(feat[k], __ldg(posedirs + k * n3 + 3 * (size_t)v + c), acc);
        p[c] = vs[3 * (size_t)v + c] + acc;
        vp_out[3 * (size_t)v + c] = p[c];
    }
    float w[GMS_FLAME_NJ];
    for (int j = 0; j < GMS_FLAME_NJ; j++) w[j] = weights[(size_t)v * GMS_FLAME_NJ + j];
    float o[3];
    for (int r = 0; r < 3; r++) {
        float T[4];
        for (int q = 0; q < 4; q++) {
            float s = 0.f;
            for (int j = 0; j < GMS_FLAME_NJ; j++) s = fmaf(w[j], A[12 * j + 4 * r + q], s);
            T[q] = s;
        }
        o[r] = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3] + t[r];
    }
    const float* e = enl + 3 * (size_t)v;
    out[3 * (size_t)v] = o[0] * e[0];
    out[3 * (size_t)v + 1] = -o[2] * e[1];
    out[3 * (size_t)v + 2] = o[1] * e[2];
    if (vgrad) { vgrad[3 * (size_t)v] = 0.f; vgrad[3 * (size_t)v + 1] = 0.f; vgrad[3 * (size_t)v + 2] = 0.f; }
}

// Backward 1: per vertex, the enlargement gradient, dL/dv_posed, and block partials of dtransl, dA (w_vj-weighted) and dfeat.
__global__ void __launch_bounds__(GMS_FLAME_VB) k_flame_skin_bwd(int V, const float* __restrict__ vp, const float* __restrict__ posedirs,
                                                                const float* __restrict__ weights, const float* __restrict__ transl,
                                                                const float* __restrict__ enl, const float* __restrict__ state,
                                                                const float* __restrict__ gout, float* __restrict__ denl,
                                                                float* __restrict__ dvp, float* __restrict__ bpart) {
    __shared__ float A[GMS_FLAME_NJ * 12], t[3];
    __shared__ float wsum[GMS_FLAME_VB / 32][GMS_FLAME_RED];
    const GmsFlameJoints* st = reinterpret_cast<const GmsFlameJoints*>(state);
    for (int k = threadIdx.x; k < GMS_FLAME_NJ * 12; k += blockDim.x) A[k] = (&st->A[0][0])[k];
    if (threadIdx.x < 3) t[threadIdx.x] = transl[threadIdx.x];
    __syncthreads();
    const int v = blockIdx.x * GMS_FLAME_VB + threadIdx.x;
    const bool live = v < V;
    const int vv = live ? v : 0;
    const size_t n3 = 3 * (size_t)V;
    float p[4], w[GMS_FLAME_NJ], d[3] = {0.f, 0.f, 0.f}, dp[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < 3; c++) p[c] = vp[3 * (size_t)vv + c];
    p[3] = 1.0f;
    for (int j = 0; j < GMS_FLAME_NJ; j++) w[j] = weights[(size_t)vv * GMS_FLAME_NJ + j];
    if (live) {
        float T[12];
        for (int k = 0; k < 12; k++) {
            float s = 0.f;
            for (int j = 0; j < GMS_FLAME_NJ; j++) s = fmaf(w[j], A[12 * j + k], s);
            T[k] = s;
        }
        float o[3];
        for (int r = 0; r < 3; r++) o[r] = T[4 * r] * p[0] + T[4 * r + 1] * p[1] + T[4 * r + 2] * p[2] + T[4 * r + 3] + t[r];
        const float* e = enl + 3 * (size_t)v;
        const float* g = gout + 3 * (size_t)v;
        denl[3 * (size_t)v] = g[0] * o[0];
        denl[3 * (size_t)v + 1] = -(g[1] * o[2]);
        denl[3 * (size_t)v + 2] = g[2] * o[1];
        d[0] = g[0] * e[0]; d[1] = g[2] * e[2]; d[2] = -(g[1] * e[1]);
        for (int q = 0; q < 3; q++) dp[q] = T[q] * d[0] + T[4 + q] * d[1] + T[8 + q] * d[2];
        for (int q = 0; q < 3; q++) dvp[3 * (size_t)v + q] = dp[q];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float r;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        r = gms_flame_warp_sum(d[c]);
        if (lane == 0) wsum[warp][c] = r;
    }
#pragma unroll
    for (int j = 0; j < GMS_FLAME_NJ; j++)
#pragma unroll
        for (int k = 0; k < 12; k++) {
            r = gms_flame_warp_sum(w[j] * d[k >> 2] * p[k & 3]);
            if (lane == 0) wsum[warp][3 + 12 * j + k] = r;
        }
    for (int k = 0; k < GMS_FLAME_NFEAT; k++) {
        const float* pd = posedirs + k * n3 + 3 * (size_t)vv;
        const float x = live ? dp[0] * __ldg(pd) + dp[1] * __ldg(pd + 1) + dp[2] * __ldg(pd + 2) : 0.f;
        r = gms_flame_warp_sum(x);
        if (lane == 0) wsum[warp][3 + 12 * GMS_FLAME_NJ + k] = r;
    }
    __syncthreads();
    if (threadIdx.x < GMS_FLAME_RED) {
        float s = 0.f;
        for (int q = 0; q < GMS_FLAME_VB / 32; q++) s += wsum[q][threadIdx.x];
        bpart[(size_t)blockIdx.x * GMS_FLAME_RED + threadIdx.x] = s;
    }
}

// Backward 2 (one block): the partials in block order, then the joint stage backward.
__global__ void k_flame_joints_bwd(int nvb, const float* __restrict__ bpart, const float* __restrict__ pose,
                                   const float* __restrict__ neck, GmsFlameParents par, const float* __restrict__ J,
                                   const float* __restrict__ state, float* __restrict__ dpose, float* __restrict__ dneck,
                                   float* __restrict__ dtransl, float* __restrict__ dJ) {
    __shared__ float red[GMS_FLAME_RED];
    if (threadIdx.x < GMS_FLAME_RED) {
        float s = 0.f;
        for (int b = 0; b < nvb; b++) s += bpart[(size_t)b * GMS_FLAME_RED + threadIdx.x];
        red[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float p[6], n[3], j[15], dp[6], dn[3], dj[15];
        for (int k = 0; k < 6; k++) p[k] = pose[k];
        for (int k = 0; k < 3; k++) n[k] = neck[k];
        for (int k = 0; k < 15; k++) j[k] = J[k];
        const GmsFlameJoints o = *reinterpret_cast<const GmsFlameJoints*>(state);
        gms_flame_joints_bwd(p, n, j, par.p, o, red + 3, red + 3 + 12 * GMS_FLAME_NJ, dp, dn, dj);
        for (int k = 0; k < 6; k++) dpose[k] = dp[k];
        for (int k = 0; k < 3; k++) { dneck[k] = dn[k]; dtransl[k] = red[k]; }
        for (int k = 0; k < 15; k++) dJ[k] = dj[k];
    }
}

#define GMS_FLAME_CB 256          // threads per column of the betas backward

// Backward 3: one block per active column b, d beta_b = shapedirs[b] . (dv_posed + J_regressor^T dJ).
__global__ void __launch_bounds__(GMS_FLAME_CB) k_flame_betas_bwd(int V, int n_shape, const float* __restrict__ shapedirs,
                                                                 const float* __restrict__ Jreg, const float* __restrict__ dvp,
                                                                 const float* __restrict__ dJ, float* __restrict__ dshape,
                                                                 float* __restrict__ dexpr) {
    __shared__ float sdJ[15], wsum[GMS_FLAME_CB / 32];
    if (threadIdx.x < 15) sdJ[threadIdx.x] = dJ[threadIdx.x];
    __syncthreads();
    const size_t n3 = 3 * (size_t)V;
    const float* row = shapedirs + (size_t)blockIdx.x * n3;
    float acc = 0.f;
    for (size_t i = threadIdx.x; i < n3; i += GMS_FLAME_CB) {
        const size_t v = i / 3;
        const int c = (int)(i - 3 * v);
        float g = dvp[i];
#pragma unroll
        for (int j = 0; j < GMS_FLAME_NJ; j++) g = fmaf(__ldg(Jreg + (size_t)j * V + v), sdJ[3 * j + c], g);
        acc = fmaf(__ldg(row + i), g, acc);
    }
    acc = gms_flame_warp_sum(acc);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int q = 0; q < GMS_FLAME_CB / 32; q++) s += wsum[q];
        const int b = blockIdx.x;
        if (b < n_shape) dshape[b] = s;
        else dexpr[b - n_shape] = s;
    }
}

#endif  // __CUDACC__
