// gms_adam.cuh -- torch.optim.Adam as fused kernels, sm_90a: k_adam over flat parameter buffers, and the SH Adam update
// with the gradient rebuilt from its factors (k_adam_sh), whose pieces the preprocess backward's fused step shares.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "gms_common.cuh"
#include "gms_preprocess.cuh"

// ---- Adam on the packed SH parameter [P,16,3] with the gradient rebuilt from its factors, dL/dSH[k][c] = basis_k(dir) * dcolor[c]:
// k_adam_sh (gms_adam_sh_factored) and the fused update of k_preprocess_bwd (gms_train_frame with sh_adam) share these pieces,
// so the two give bit-identical p, m and v.

// torch.optim.Adam's constants: (1 - beta), lr / (1 - beta1^t), sqrt(1 - beta2^t) are formed in double on the host and rounded
// once (torch: Python floats).  The DC coefficient uses lr_dc, the other 15 lr_rest.
struct AdamShConst { float lr_dc, lr_rest, beta1, beta2, omb1, omb2, eps, bc2_sqrt; };

static AdamShConst adam_sh_const(double lr_dc, double lr_rest, double beta1, double beta2, double eps, int step) {
    AdamShConst c;
    const double bc1 = 1.0 - pow(beta1, (double)step);
    c.lr_dc = (float)(lr_dc / bc1); c.lr_rest = (float)(lr_rest / bc1);
    c.beta1 = (float)beta1; c.beta2 = (float)beta2; c.eps = (float)eps;
    c.omb1 = (float)(1.0 - beta1); c.omb2 = (float)(1.0 - beta2);
    c.bc2_sqrt = (float)sqrt(1.0 - pow(beta2, (double)step));
    return c;
}

// SH basis at normalize(xyz - campos) (same direction arithmetic as gms_sh_backward), zeros above degree D.
__device__ __forceinline__ void sh_grad_basis(int D, float mx, float my, float mz, const float* cp, float B[16]) {
    float dx = mx - __ldg(cp), dy = my - __ldg(cp + 1), dz = mz - __ldg(cp + 2);
    const float len = GMS_SQRTP(dx * dx + dy * dy + dz * dz);
    dx = GMS_DIVP(dx, len); dy = GMS_DIVP(dy, len); dz = GMS_DIVP(dz, len);
#pragma unroll
    for (int k = 0; k < 16; k++) B[k] = 0.f;
    gms_sh_basis(D, dx, dy, dz, B);
}

// One float4 of a packed row (elements 4c .. 4c+3 of the 48) through the update.  The default uses the branch-free correctly-
// rounded division / square root of gms_common.cuh (GMS_DIVN / GMS_SQRTN): the three slow-path branches per element of
// `sqrtf(v) / bc + eps` and `m / denom` serialised the twelve MUFU chains of a float4 (stalled on fixed-latency dependencies,
// not on memory).  Adam's divisors are normal numbers (bias correction; sqrt(v)/bc + eps >= eps); tiny / denormal second
// moments are handled inside gms_sqrt_rn_normal; a denormal numerator m only loses bits below 1e-38.
// Every multiply-add is spelled out: left to the compiler, whether `p - step * q` becomes one FFMA or FMUL + FADD depends on
// the code around it, and the two kernels must round alike.  The explicit forms are the ones k_adam_sh was compiled to.
template <bool IEEE_CALLS>
__device__ __forceinline__ void adam_sh_update4(const AdamShConst& a, int c, const float gv[4], float pv[4], float mv[4], float vv[4]) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const float step = (4 * c + k < 3) ? a.lr_dc : a.lr_rest;       // coefficient 0 = the DC term (f_dc), the rest f_rest
        mv[k] = __fmaf_rn(a.beta1, mv[k], __fmul_rn(a.omb1, gv[k]));
        vv[k] = __fmaf_rn(a.beta2, vv[k], __fmul_rn(__fmul_rn(a.omb2, gv[k]), gv[k]));
        if (IEEE_CALLS) {       // A/B arm (option adam_sh_ieee=1): nvcc's own sqrtf and `/` with their slow-path branches
            const float denom = __fadd_rn(sqrtf(vv[k]) / a.bc2_sqrt, a.eps);
            pv[k] = __fmaf_rn(-step, mv[k] / denom, pv[k]);
        } else {
            const float denom = __fadd_rn(gms_div_rn_normal(gms_sqrt_rn_normal(vv[k]), a.bc2_sqrt), a.eps);
            pv[k] = __fmaf_rn(-step, gms_div_rn_normal(mv[k], denom), pv[k]);
        }
    }
}

// ------------------------------------------------------------------------------------------ fused Adam
// torch.optim.Adam(lr per group, betas, eps=1e-15) of gaussian_mesh_model.py:171-183 over ONE flat parameter buffer:
// p, g, m, v are flat fp32 arrays; segments carry the per-group learning rates (feature segment: lr0 for the DC
// coefficient, lr1 for the rest).  The gradient is consumed and zeroed in the same pass (no separate memset).
struct AdamSeg { long long end; float lr0, lr1; int inner, period; };     // lr0/lr1: step sizes lr / (1 - beta1^t)
struct AdamArgs { long long n; long long offset; float* p; float* g; float* m; float* v; int nseg; AdamSeg seg[8];
                  float beta1, beta2, omb1, omb2, eps, bc2_sqrt; int zero_grad; long long zero_end; };

// One thread = 4 consecutive elements.  Segment boundaries are looked up once per thread; the DC/rest learning-rate
// phase of the packed SH segment is carried incrementally (one 32-bit division per thread instead of a 64-bit
// division per element).  Threads whose 4 elements straddle a segment end (never the case for FlatAdam's 64-float
// padded segments) or the end of the buffer take the per-element path.
__device__ __forceinline__ void adam_locate(const AdamArgs& a, long long i, int& sidx, long long& start) {
    sidx = 0; start = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) if (q < a.nseg - 1 && i >= a.seg[q].end) { sidx = q + 1; start = a.seg[q].end; }
}

// torch.optim.Adam's arithmetic: the constants (1 - beta), lr / (1 - beta1^t), sqrt(1 - beta2^t) are formed in double
// on the host and rounded once (torch: Python floats), `step` is the step size lr / bias_correction1.
__device__ __forceinline__ void adam_update(const AdamArgs& a, float step, float g, float& p, float& m, float& v) {
    m = a.beta1 * m + a.omb1 * g;
    v = a.beta2 * v + a.omb2 * g * g;
    const float denom = sqrtf(v) / a.bc2_sqrt + a.eps;
    p = p - step * (m / denom);
}

__global__ void __launch_bounds__(256) k_adam(AdamArgs a) {
    const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i4 >= a.n) return;
    const long long gi = a.offset + i4;          // flat index: p/g/m/v point at element `offset` of the flat buffers
    int sidx; long long start;
    adam_locate(a, gi, sidx, start);
    const AdamSeg sg = a.seg[sidx];
    const bool full = i4 + 4 <= a.n && (sidx == a.nseg - 1 || gi + 4 <= sg.end);
    if (full) {
        const float4 P4 = *reinterpret_cast<const float4*>(a.p + i4), G4 = *reinterpret_cast<const float4*>(a.g + i4);
        const float4 M4 = *reinterpret_cast<const float4*>(a.m + i4), V4 = *reinterpret_cast<const float4*>(a.v + i4);
        float pv[4] = {P4.x, P4.y, P4.z, P4.w}, mv[4] = {M4.x, M4.y, M4.z, M4.w}, vv[4] = {V4.x, V4.y, V4.z, V4.w};
        const float gv[4] = {G4.x, G4.y, G4.z, G4.w};
        if (sg.period > 0) {
            const unsigned long long rel = (unsigned long long)(gi - start);
            unsigned q, r;                         // rel = q * inner + r
            if (rel < 0xffffffffull) { q = (unsigned)rel / (unsigned)sg.inner; r = (unsigned)rel - q * (unsigned)sg.inner; }
            else { const unsigned long long q64 = rel / (unsigned)sg.inner; r = (unsigned)(rel - q64 * (unsigned)sg.inner); q = (unsigned)(q64 % (unsigned)sg.period); }
            unsigned phase = q % (unsigned)sg.period;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                adam_update(a, phase == 0 ? sg.lr0 : sg.lr1, gv[k], pv[k], mv[k], vv[k]);
                if (++r == (unsigned)sg.inner) { r = 0; if (++phase == (unsigned)sg.period) phase = 0; }
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) adam_update(a, sg.lr0, gv[k], pv[k], mv[k], vv[k]);
        }
        *reinterpret_cast<float4*>(a.p + i4) = make_float4(pv[0], pv[1], pv[2], pv[3]);
        *reinterpret_cast<float4*>(a.m + i4) = make_float4(mv[0], mv[1], mv[2], mv[3]);
        *reinterpret_cast<float4*>(a.v + i4) = make_float4(vv[0], vv[1], vv[2], vv[3]);
        if (a.zero_grad == 1 || (a.zero_grad == 2 && gi + 4 <= a.zero_end))
            *reinterpret_cast<float4*>(a.g + i4) = make_float4(0.f, 0.f, 0.f, 0.f);
        else if (a.zero_grad == 2 && gi < a.zero_end)
            for (int k = 0; k < 4; k++) if (gi + k < a.zero_end) a.g[i4 + k] = 0.f;
        return;
    }
    for (int k = 0; k < 4; k++) {
        if (i4 + k >= a.n) break;
        const long long i = gi + k;
        int sx; long long st;
        adam_locate(a, i, sx, st);
        const AdamSeg s1 = a.seg[sx];
        float lr = s1.lr0;
        if (s1.period > 0) lr = (((i - st) / s1.inner) % s1.period == 0) ? s1.lr0 : s1.lr1;
        float pv = a.p[i4 + k], mv = a.m[i4 + k], vv = a.v[i4 + k];
        adam_update(a, lr, a.g[i4 + k], pv, mv, vv);
        a.p[i4 + k] = pv; a.m[i4 + k] = mv; a.v[i4 + k] = vv;
        if (a.zero_grad == 1 || (a.zero_grad == 2 && i < a.zero_end)) a.g[i4 + k] = 0.f;
    }
}

// Adam on the packed SH parameter with the gradient rebuilt on the fly from its factors (gms_adam_sh_factored):
//   dL/dSH_i[k][c] = (1/R) * sum_r basis_k(normalize(xyz_i - campos_r)) * dcolor_r[i][c]
// -- per camera the SH gradient of a Gaussian is the outer product of the SH basis at its view direction and the (clamp-
// masked) colour gradient, so R ranks exchange 12 B per Gaussian instead of reducing 192 B, and the 192 B/Gaussian gradient
// rows are never written or read.  Same update arithmetic as k_adam (torch.optim.Adam).
struct AdamShArgs {
    int P, D, R; long long slot;     // slot = floats between the ranks' exchange slots ([3P colour gradients | 3 campos | pad])
    const float* xyz; const float* xbuf;
    float* p; float* m; float* v;
    float scale;
    AdamShConst c;
};

template <bool IEEE_CALLS>
__global__ void __launch_bounds__(128, 6) k_adam_sh(AdamShArgs a) {
    // A warp handles 32 Gaussians.  Phase A: lane i rebuilds Gaussian i's 48 gradient values from the R colour gradients
    // (direction, SH basis, 48 FMAs per rank -- the ranks' loads are issued one rank ahead) into a shared-memory tile (row
    // stride 49: conflict-free).  Phase B: the warp walks the tile row-major with coalesced 128-bit accesses to p / m / v --
    // the loads of the next 32 float4s are in flight while the current ones are updated -- and applies torch.optim.Adam's update.
    constexpr int STRIDE = 49;
    __shared__ float s_g[4][32 * STRIDE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i0 = (blockIdx.x * 4 + warp) * 32, i = i0 + lane;
    if (i0 >= a.P) return;
    float* tile = s_g[warp];
    const size_t base4 = (size_t)i0 * 12;      // float4 index of the warp's first row
    const float4* p4 = reinterpret_cast<const float4*>(a.p) + base4;
    const float4* m4 = reinterpret_cast<const float4*>(a.m) + base4;
    const float4* v4 = reinterpret_cast<const float4*>(a.v) + base4;
    const int nrow = min(32, a.P - i0), n4 = 12 * nrow;
    // phase B's streams run two 32-float4 groups ahead of the update (3 KB per warp in flight); the first two are issued
    // here, before phase A
    constexpr int AHEAD = 2;
    float4 Pb[AHEAD + 1], Mb[AHEAD + 1], Vb[AHEAD + 1];
#pragma unroll
    for (int q = 0; q < AHEAD; q++) {
        Pb[q] = Mb[q] = Vb[q] = make_float4(0, 0, 0, 0);
        if (q * 32 + lane < n4) { Pb[q] = p4[q * 32 + lane]; Mb[q] = m4[q * 32 + lane]; Vb[q] = v4[q * 32 + lane]; }
    }
    {   // phase A accumulates straight into the lane's tile row (no 48 accumulator registers: 8 CTAs per SM instead of 4)
        float* row = tile + lane * STRIDE;
        bool first = true;
        if (i < a.P) {
            const float mx = a.xyz[3 * i], my = a.xyz[3 * i + 1], mz = a.xyz[3 * i + 2];
            float n0 = a.xbuf[3 * i], n1 = a.xbuf[3 * i + 1], n2 = a.xbuf[3 * i + 2];
            for (int r = 0; r < a.R; r++) {
                const float g0 = n0 * a.scale, g1 = n1 * a.scale, g2 = n2 * a.scale;
                if (r + 1 < a.R) { const float* nx = a.xbuf + (size_t)(r + 1) * a.slot + 3 * i; n0 = nx[0]; n1 = nx[1]; n2 = nx[2]; }
                if (g0 == 0.f && g1 == 0.f && g2 == 0.f) continue;      // culled / unblended / clamped at that camera
                float B[16];
                sh_grad_basis(a.D, mx, my, mz, a.xbuf + (size_t)r * a.slot + 3 * (size_t)a.P, B);
                if (first) {
#pragma unroll
                    for (int k = 0; k < 16; k++) { row[3 * k] = B[k] * g0; row[3 * k + 1] = B[k] * g1; row[3 * k + 2] = B[k] * g2; }
                    first = false;
                } else {
#pragma unroll
                    for (int k = 0; k < 16; k++) { row[3 * k] += B[k] * g0; row[3 * k + 1] += B[k] * g1; row[3 * k + 2] += B[k] * g2; }
                }
            }
        }
        if (first) {
#pragma unroll
            for (int k = 0; k < 48; k++) row[k] = 0.f;
        }
    }
    __syncwarp();
    float4* po = reinterpret_cast<float4*>(a.p) + base4;
    float4* mo = reinterpret_cast<float4*>(a.m) + base4;
    float4* vo = reinterpret_cast<float4*>(a.v) + base4;
#pragma unroll
    for (int it = 0; it < 12; it++) {
        const int j = it * 32 + lane;
        if (it + AHEAD < 12) {
            const int jn = j + AHEAD * 32, sl = (it + AHEAD) % (AHEAD + 1);
            Pb[sl] = Mb[sl] = Vb[sl] = make_float4(0, 0, 0, 0);
            if (jn < n4) { Pb[sl] = p4[jn]; Mb[sl] = m4[jn]; Vb[sl] = v4[jn]; }
        }
        const float4 Pc = Pb[it % (AHEAD + 1)], Mc = Mb[it % (AHEAD + 1)], Vc = Vb[it % (AHEAD + 1)];
        if (j < n4) {
            const int r = j / 12, c = j - r * 12;
            const float* gq = tile + r * STRIDE + 4 * c;
            const float gv[4] = {gq[0], gq[1], gq[2], gq[3]};
            float pv[4] = {Pc.x, Pc.y, Pc.z, Pc.w}, mv[4] = {Mc.x, Mc.y, Mc.z, Mc.w}, vv[4] = {Vc.x, Vc.y, Vc.z, Vc.w};
            adam_sh_update4<IEEE_CALLS>(a.c, c, gv, pv, mv, vv);
            po[j] = make_float4(pv[0], pv[1], pv[2], pv[3]);
            mo[j] = make_float4(mv[0], mv[1], mv[2], mv[3]);
            vo[j] = make_float4(vv[0], vv[1], vv[2], vv[3]);
        }
    }
}
