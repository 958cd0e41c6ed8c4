// gms_expand.cuh -- per-face maths of the mesh -> Gaussian expansion, forward and hand-derived backward.
// Host+device (see gms_common.cuh).  One thread owns one face: the face frame and its quaternion are
// computed ONCE per face (the reference recomputes them for each of the K splats of a face).
//
// Replaces (reference, pure PyTorch, ~45 ATen kernels per call + their autograd):
//   GaussianMeshModel.update_alpha / _calc_xyz      games/mesh_splatting/scene/gaussian_mesh_model.py:153-169, 86-101
//   GaussianMeshModel.prepare_scaling_rot           games/mesh_splatting/scene/gaussian_mesh_model.py:103-151
//   rot_to_quat_batch / _sqrt_positive_part / standardize_quaternion      utils/general_utils.py:19-96
//   get_scaling = exp, get_rotation = normalize (optional fused outputs)  scene/gaussian_model.py:95-101
#pragma once
#include "gms_common.cuh"
#include "../../include/gms_b200.h"

struct GmsFrame {
    float v0[3], v1[3], v2[3];   // rotation COLUMNS
    float n[3], nn;              // un-normalised normal and its norm
    float a1[3], na1;            // t1 - mean, |a1|
    float a2[3];                 // t2 - mean
    float u[3], nu;              // Gram-Schmidt residual and its norm
    float d0, d1;                // a2.v0, a2.v1
    float s[3];                  // (eps, s1, s2)
};

GMS_HD float gms_norm3(const float* v) { return GMS_SQRTN(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
GMS_HD float gms_dotv(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// t = [t0 | t1 | t2] (9 floats)
GMS_HD void gms_face_frame(const float* t, float eps, GmsFrame& f) {
    const float* t0 = t; const float* t1 = t + 3; const float* t2 = t + 6;
    float e1[3], e2[3], m[3];
#pragma unroll
    for (int i = 0; i < 3; i++) { e1[i] = t1[i] - t0[i]; e2[i] = t2[i] - t0[i]; m[i] = GMS_DIVN(t0[i] + t1[i] + t2[i], 3.0f); }
    f.n[0] = e1[1] * e2[2] - e1[2] * e2[1];
    f.n[1] = e1[2] * e2[0] - e1[0] * e2[2];
    f.n[2] = e1[0] * e2[1] - e1[1] * e2[0];
    f.nn = gms_norm3(f.n);
    const float inn = GMS_DIVN(1.0f, f.nn + eps);
#pragma unroll
    for (int i = 0; i < 3; i++) { f.v0[i] = f.n[i] * inn; f.a1[i] = t1[i] - m[i]; f.a2[i] = t2[i] - m[i]; }
    f.na1 = gms_norm3(f.a1);
    const float l1 = f.na1 + eps;
#pragma unroll
    for (int i = 0; i < 3; i++) f.v1[i] = GMS_DIVN(f.a1[i], l1);
    f.d0 = gms_dotv(f.a2, f.v0);
    f.d1 = gms_dotv(f.a2, f.v1);
#pragma unroll
    for (int i = 0; i < 3; i++) f.u[i] = f.a2[i] - f.d0 * f.v0[i] - f.d1 * f.v1[i];
    f.nu = gms_norm3(f.u);
    const float lu = f.nu + eps;
#pragma unroll
    for (int i = 0; i < 3; i++) f.v2[i] = GMS_DIVN(f.u[i], lu);
    f.s[0] = eps;
    f.s[1] = l1 / 2.0f;
    f.s[2] = gms_dotv(f.a2, f.v2) / 2.0f;
}

struct GmsQuatAux { int sel; float sgn; float qa; float D; float cand[4]; };

// pytorch3d matrix_to_quaternion on R = [v0|v1|v2] (columns); q = (w,x,y,z) with w >= 0
GMS_HD void gms_frame_quat(const GmsFrame& f, float* q, GmsQuatAux& ax) {
    const float m00 = f.v0[0], m01 = f.v1[0], m02 = f.v2[0];
    const float m10 = f.v0[1], m11 = f.v1[1], m12 = f.v2[1];
    const float m20 = f.v0[2], m21 = f.v1[2], m22 = f.v2[2];
    float x[4] = {1.0f + m00 + m11 + m22, 1.0f + m00 - m11 - m22, 1.0f - m00 + m11 - m22, 1.0f - m00 - m11 + m22};
    float qa[4];
#pragma unroll
    for (int i = 0; i < 4; i++) qa[i] = x[i] > 0.f ? GMS_SQRTN(x[i]) : 0.f;
    int sel = 0;
#pragma unroll
    for (int i = 1; i < 4; i++) if (qa[i] > qa[sel]) sel = i;   // first maximum, like torch.argmax
    float c[4];
    const float qq = qa[sel] * qa[sel];
    if (sel == 0)      { c[0] = qq;        c[1] = m21 - m12; c[2] = m02 - m20; c[3] = m10 - m01; }
    else if (sel == 1) { c[0] = m21 - m12; c[1] = qq;        c[2] = m10 + m01; c[3] = m02 + m20; }
    else if (sel == 2) { c[0] = m02 - m20; c[1] = m10 + m01; c[2] = qq;        c[3] = m12 + m21; }
    else               { c[0] = m10 - m01; c[1] = m20 + m02; c[2] = m21 + m12; c[3] = qq; }
    const float D = 2.0f * fmaxf(qa[sel], 0.1f);
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; i++) o[i] = GMS_DIVN(c[i], D);        // D >= 0.2
    const float sgn = o[0] < 0.f ? -1.f : 1.f;
#pragma unroll
    for (int i = 0; i < 4; i++) { q[i] = sgn * o[i]; ax.cand[i] = c[i]; }
    ax.sel = sel; ax.sgn = sgn; ax.qa = qa[sel]; ax.D = D;
}

// gradient of the quaternion w.r.t. the three frame columns
GMS_HD void gms_frame_quat_backward(const GmsQuatAux& ax, const float* dq, float* dv0, float* dv1, float* dv2) {
    float dc[4]; float dD = 0.f;
#pragma unroll
    for (int i = 0; i < 4; i++) { dc[i] = GMS_DIVN(ax.sgn * dq[i], ax.D); dD -= GMS_DIVN(ax.sgn * dq[i] * ax.cand[i], ax.D * ax.D); }
    // d x_sel : cand[sel] = qa^2 = x (x > 0) ; D = 2*max(qa, 0.1)
    float dx = 0.f;
    if (ax.qa > 0.f) {
        dx = dc[ax.sel];
        if (ax.qa > 0.1f) dx += GMS_DIVN(dD, ax.qa);        // dD * dD/dqa * dqa/dx = dD * 2 * 1/(2 qa)
    }
    float dm[9];
#pragma unroll
    for (int i = 0; i < 9; i++) dm[i] = 0.f;
    // x_sel = 1 + s0*m00 + s1*m11 + s2*m22
    const float s00 = (ax.sel == 0 || ax.sel == 1) ? 1.f : -1.f;
    const float s11 = (ax.sel == 0 || ax.sel == 2) ? 1.f : -1.f;
    const float s22 = (ax.sel == 0 || ax.sel == 3) ? 1.f : -1.f;
    dm[0] += s00 * dx; dm[4] += s11 * dx; dm[8] += s22 * dx;
    // off-diagonal candidates; index dm[3*a+b] = m_ab
    if (ax.sel == 0) {
        dm[7] += dc[1]; dm[5] -= dc[1];   // m21 - m12
        dm[2] += dc[2]; dm[6] -= dc[2];   // m02 - m20
        dm[3] += dc[3]; dm[1] -= dc[3];   // m10 - m01
    } else if (ax.sel == 1) {
        dm[7] += dc[0]; dm[5] -= dc[0];   // m21 - m12
        dm[3] += dc[2]; dm[1] += dc[2];   // m10 + m01
        dm[2] += dc[3]; dm[6] += dc[3];   // m02 + m20
    } else if (ax.sel == 2) {
        dm[2] += dc[0]; dm[6] -= dc[0];   // m02 - m20
        dm[3] += dc[1]; dm[1] += dc[1];   // m10 + m01
        dm[5] += dc[3]; dm[7] += dc[3];   // m12 + m21
    } else {
        dm[3] += dc[0]; dm[1] -= dc[0];   // m10 - m01
        dm[6] += dc[1]; dm[2] += dc[1];   // m20 + m02
        dm[7] += dc[2]; dm[5] += dc[2];   // m21 + m12
    }
    // m_ab = v_b[a]
#pragma unroll
    for (int a = 0; a < 3; a++) { dv0[a] += dm[3 * a + 0]; dv1[a] += dm[3 * a + 1]; dv2[a] += dm[3 * a + 2]; }
}

// Back-propagate (dv0, dv1, dv2, ds1, ds2) through the face frame to the triangle corners; dt += ...
GMS_HD void gms_face_frame_backward(const float* t, float eps, const GmsFrame& f, float* dv0, float* dv1, float* dv2,
                                    float ds1, float ds2, float* dt) {
    const float* t0 = t; const float* t1 = t + 3; const float* t2 = t + 6;
    float da1[3] = {0.f, 0.f, 0.f}, da2[3] = {0.f, 0.f, 0.f};
    // s2 = (a2 . v2) / 2
#pragma unroll
    for (int i = 0; i < 3; i++) { da2[i] += 0.5f * ds2 * f.v2[i]; dv2[i] += 0.5f * ds2 * f.a2[i]; }
    // v2 = u / (|u| + eps)
    const float lu = f.nu + eps;
    float du[3];
    {
        const float k = f.nu > 0.f ? gms_dotv(dv2, f.u) / (f.nu * lu * lu) : 0.f;
#pragma unroll
        for (int i = 0; i < 3; i++) du[i] = GMS_DIVN(dv2[i], lu) - k * f.u[i];
    }
    // u = a2 - (a2.v0) v0 - (a2.v1) v1
    {
        const float p0 = gms_dotv(du, f.v0), p1 = gms_dotv(du, f.v1);
#pragma unroll
        for (int i = 0; i < 3; i++) {
            da2[i] += du[i] - p0 * f.v0[i] - p1 * f.v1[i];
            dv0[i] += -p0 * f.a2[i] - f.d0 * du[i];
            dv1[i] += -p1 * f.a2[i] - f.d1 * du[i];
        }
    }
    // v1 = a1 / l1 ; l1 = |a1| + eps ; s1 = l1 / 2
    {
        const float l1 = f.na1 + eps;
        const float dl1 = 0.5f * ds1 - GMS_DIVN(gms_dotv(dv1, f.a1), l1 * l1);      // l1 >= eps: l1^2 >= 1e-16
        const float k = f.na1 > 0.f ? dl1 / f.na1 : 0.f;
#pragma unroll
        for (int i = 0; i < 3; i++) da1[i] += GMS_DIVN(dv1[i], l1) + k * f.a1[i];
    }
    // a1 = t1 - m ; a2 = t2 - m ; m = (t0+t1+t2)/3
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float dm = GMS_DIVN(-(da1[i] + da2[i]), 3.0f);
        dt[i] += dm; dt[3 + i] += da1[i] + dm; dt[6 + i] += da2[i] + dm;
    }
    // v0 = n / (|n| + eps) ; n = e1 x e2
    {
        const float ln = f.nn + eps;
        const float k = f.nn > 0.f ? gms_dotv(dv0, f.n) / (f.nn * ln * ln) : 0.f;
        float dn[3], e1[3], e2[3];
#pragma unroll
        for (int i = 0; i < 3; i++) { dn[i] = GMS_DIVN(dv0[i], ln) - k * f.n[i]; e1[i] = t1[i] - t0[i]; e2[i] = t2[i] - t0[i]; }
        const float de1[3] = {e2[1] * dn[2] - e2[2] * dn[1], e2[2] * dn[0] - e2[0] * dn[2], e2[0] * dn[1] - e2[1] * dn[0]};
        const float de2[3] = {dn[1] * e1[2] - dn[2] * e1[1], dn[2] * e1[0] - dn[0] * e1[2], dn[0] * e1[1] - dn[1] * e1[0]};
#pragma unroll
        for (int i = 0; i < 3; i++) { dt[3 + i] += de1[i]; dt[6 + i] += de2[i]; dt[i] -= de1[i] + de2[i]; }
    }
}

// ---- whole-face forward / backward (called by k_expand_fwd / k_expand_bwd, and by tests/hostshim on the CPU)
#if defined(__CUDA_ARCH__)
#define GMS_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#else
#define GMS_ATOMIC_ADD(p, v) (*(p) += (v))
#endif

// Barycentric weights of one splat from its three raw parameters (gms_expand_args.alpha_activation):
//   GMS_ALPHA_RELU     r_j = relu(x_j) + 1e-8, alpha_j = r_j / sum r   (GaussianMeshModel.update_alpha, gaussian_mesh_model.py:166-167)
//   GMS_ALPHA_SOFTMAX  alpha = softmax(x)                               (GaussianFlameModel.update_alpha_func, gaussian_flame_model.py:34,195)
// The softmax subtracts the row maximum first, so logits far above 88 cannot overflow expf: e_j = exp(x_j - m) lies in
// (0, 1] and the largest is exactly 1, so s = (e0 + e1) + e2 lies in [1, 3].

// `f` indexes the per-FACE arrays (faces / triangles_in / triangles); `fl` indexes the per-GAUSSIAN streams (alpha_raw,
// scale_raw and every output row): fl == f when they are the caller's arrays, fl == the face's slot in the block when the
// kernel has redirected those pointers to its shared-memory staging buffers (the staged k_expand_fwd).
// A face is read, its frame and quaternion formed once (gms_expand_face_load / gms_expand_face_frame), then every splat is one call of
// gms_expand_splat_fwd / gms_expand_splat_bwd: the per-thread kernels loop over the face's K splats, the wide kernels
// (k_expand_wide_*) spread them over a warp's lanes.  Either way each splat's arithmetic is the same sequence of operations.
struct GmsFaceState {
    float t[9];
    int64_t vi[3];
    GmsFrame fr;
    float q[4];
    GmsQuatAux ax;
    float qnorm, qn;
};

GMS_HD void gms_expand_face_load(const gms_expand_args& a, int f, GmsFaceState& s) {
    s.vi[0] = s.vi[1] = s.vi[2] = 0;
    if (a.triangles_in) {
#pragma unroll
        for (int k = 0; k < 9; k++) s.t[k] = a.triangles_in[9 * (size_t)f + k];
    } else {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            s.vi[c] = a.faces[3 * (size_t)f + c];
            s.t[3 * c] = a.vertices[3 * s.vi[c]]; s.t[3 * c + 1] = a.vertices[3 * s.vi[c] + 1]; s.t[3 * c + 2] = a.vertices[3 * s.vi[c] + 2];
        }
    }
}

GMS_HD void gms_expand_face_frame(const gms_expand_args& a, GmsFaceState& s) {
    gms_face_frame(s.t, a.eps, s.fr);
    gms_frame_quat(s.fr, s.q, s.ax);
    s.qnorm = GMS_SQRTN(s.q[0] * s.q[0] + s.q[1] * s.q[1] + s.q[2] * s.q[2] + s.q[3] * s.q[3]);
    s.qn = fmaxf(s.qnorm, 1e-12f);
}

template <int ACT>
GMS_HD void gms_alpha_fwd(float x0, float x1, float x2, float& al0, float& al1, float& al2) {
    if constexpr (ACT == GMS_ALPHA_SOFTMAX) {
        const float m = fmaxf(fmaxf(x0, x1), x2);
        const float e0 = expf(x0 - m), e1 = expf(x1 - m), e2 = expf(x2 - m);
        const float s = (e0 + e1) + e2;                                                       // s in [1, 3]
        al0 = GMS_DIVN(e0, s); al1 = GMS_DIVN(e1, s); al2 = GMS_DIVN(e2, s);
    } else {
        const float r0 = fmaxf(x0, 0.f) + 1e-8f, r1 = fmaxf(x1, 0.f) + 1e-8f, r2 = fmaxf(x2, 0.f) + 1e-8f;
        const float S = r0 + r1 + r2;
        al0 = GMS_DIVN(r0, S); al1 = GMS_DIVN(r1, S); al2 = GMS_DIVN(r2, S);        // S >= 3e-8
    }
}

// Splat p of a face whose frame is in `s`.
template <int ACT>
GMS_HD void gms_expand_splat_fwd(const gms_expand_args& a, const GmsFaceState& s, size_t p) {
    const float* t = s.t;
    float al0, al1, al2;
    gms_alpha_fwd<ACT>(a.alpha_raw[3 * p], a.alpha_raw[3 * p + 1], a.alpha_raw[3 * p + 2], al0, al1, al2);
    if (a.alpha) { a.alpha[3 * p] = al0; a.alpha[3 * p + 1] = al1; a.alpha[3 * p + 2] = al2; }
    if (a.xyz) {
#pragma unroll
        for (int c = 0; c < 3; c++) a.xyz[3 * p + c] = al0 * t[c] + al1 * t[3 + c] + al2 * t[6 + c];
    }
    const float cs = a.scale_raw[p];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float inner = fmaxf(cs * s.fr.s[c], 0.f) + a.eps;
        if (a.scaling_log) a.scaling_log[3 * p + c] = logf(inner);
        if (a.scaling_act) a.scaling_act[3 * p + c] = expf(logf(inner));
    }
    const float* q = s.q;
    const float qn = s.qn;
    if (a.rotation_raw) { float* o = a.rotation_raw + 4 * p; o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3]; }
    if (a.rotation_act) { float* o = a.rotation_act + 4 * p; o[0] = GMS_DIVN(q[0], qn); o[1] = GMS_DIVN(q[1], qn); o[2] = GMS_DIVN(q[2], qn); o[3] = GMS_DIVN(q[3], qn); }
}

template <int ACT>
GMS_HD void gms_expand_face_fwd_act(const gms_expand_args& a, int f, int fl) {
    GmsFaceState s;
    gms_expand_face_load(a, f, s);
    if (a.triangles) {
#pragma unroll
        for (int k = 0; k < 9; k++) a.triangles[9 * (size_t)f + k] = s.t[k];
    }
    gms_expand_face_frame(a, s);
    for (int k = 0; k < a.K; k++) gms_expand_splat_fwd<ACT>(a, s, (size_t)fl * a.K + k);
}

// The backward of splat p: writes its dL/d_alpha and dL/d_scale rows and ADDS its share of the face's corner, quaternion
// and in-plane scale gradients to dt / dq / ds1 / ds2.
template <int ACT>
GMS_HD void gms_expand_splat_bwd(const gms_expand_args& a, const gms_expand_grads& g, const GmsFaceState& s, size_t p,
                                 float* dt, float* dq, float& ds1, float& ds2) {
    const float* t = s.t;
    const float* q = s.q;
    const float qnorm = s.qnorm, qn = s.qn;
    // --- xyz = alpha @ triangle
    float dx[3] = {0.f, 0.f, 0.f};
    if (g.dL_dxyz) { dx[0] = g.dL_dxyz[3 * p]; dx[1] = g.dL_dxyz[3 * p + 1]; dx[2] = g.dL_dxyz[3 * p + 2]; }
    const float ar[3] = {a.alpha_raw[3 * p], a.alpha_raw[3 * p + 1], a.alpha_raw[3 * p + 2]};
    float al[3];
    gms_alpha_fwd<ACT>(ar[0], ar[1], ar[2], al[0], al[1], al[2]);
    float dal[3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        dal[j] = dx[0] * t[3 * j] + dx[1] * t[3 * j + 1] + dx[2] * t[3 * j + 2];
#pragma unroll
        for (int c = 0; c < 3; c++) dt[3 * j + c] += al[j] * dx[c];
    }
    const float dsum = dal[0] * al[0] + dal[1] * al[1] + dal[2] * al[2];
    if (g.dL_dalpha_raw) {
        if constexpr (ACT == GMS_ALPHA_SOFTMAX) {
#pragma unroll
            for (int j = 0; j < 3; j++) g.dL_dalpha_raw[3 * p + j] = al[j] * (dal[j] - dsum);
        } else {
            const float S = (fmaxf(ar[0], 0.f) + 1e-8f) + (fmaxf(ar[1], 0.f) + 1e-8f) + (fmaxf(ar[2], 0.f) + 1e-8f);
#pragma unroll
            for (int j = 0; j < 3; j++) g.dL_dalpha_raw[3 * p + j] = ar[j] > 0.f ? GMS_DIVN(dal[j] - dsum, S) : 0.f;
        }
    }
    // --- scaling
    const float cs = a.scale_raw[p];
    float dcs = 0.f;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float gl = g.dL_dscaling_log ? g.dL_dscaling_log[3 * p + c] : 0.f;
        const float prod = cs * s.fr.s[c];
        const float inner = fmaxf(prod, 0.f) + a.eps;
        if (g.dL_dscaling_act) gl += g.dL_dscaling_act[3 * p + c] * expf(logf(inner));
        const float dprod = prod > 0.f ? GMS_DIVN(gl, inner) : 0.f;       // inner >= eps
        dcs += dprod * s.fr.s[c];
        if (c == 1) ds1 += dprod * cs;
        if (c == 2) ds2 += dprod * cs;
    }
    if (g.dL_dscale_raw) g.dL_dscale_raw[p] = dcs;
    // --- rotation (same quaternion for the K splats of the face: sum the incoming rows)
    if (g.dL_drotation_raw) {
        const float* d = g.dL_drotation_raw + 4 * p;
        dq[0] += d[0]; dq[1] += d[1]; dq[2] += d[2]; dq[3] += d[3];
    }
    if (g.dL_drotation_act) {
        const float* dp = g.dL_drotation_act + 4 * p;
        const float d_x = dp[0], d_y = dp[1], d_z = dp[2], d_w = dp[3];
        if (qnorm >= 1e-12f) {
            const float u[4] = {GMS_DIVN(q[0], qn), GMS_DIVN(q[1], qn), GMS_DIVN(q[2], qn), GMS_DIVN(q[3], qn)};       // qn >= 1e-12
            const float dd = d_x * u[0] + d_y * u[1] + d_z * u[2] + d_w * u[3];
            dq[0] += GMS_DIVN(d_x - u[0] * dd, qn); dq[1] += GMS_DIVN(d_y - u[1] * dd, qn);
            dq[2] += GMS_DIVN(d_z - u[2] * dd, qn); dq[3] += GMS_DIVN(d_w - u[3] * dd, qn);
        } else {
            dq[0] += GMS_DIVN(d_x, qn); dq[1] += GMS_DIVN(d_y, qn); dq[2] += GMS_DIVN(d_z, qn); dq[3] += GMS_DIVN(d_w, qn);
        }
    }
}

// The face's share once every splat's has been summed: through the quaternion and the frame to the corners, then
// dL_dtriangles and the vertex atomics.
GMS_HD void gms_expand_face_bwd_tail(const gms_expand_args& a, const gms_expand_grads& g, const GmsFaceState& s, int f, float* dt,
                                     const float* dq, float ds1, float ds2) {
    float dv0[3] = {0.f, 0.f, 0.f}, dv1[3] = {0.f, 0.f, 0.f}, dv2[3] = {0.f, 0.f, 0.f};
    gms_frame_quat_backward(s.ax, dq, dv0, dv1, dv2);
    gms_face_frame_backward(s.t, a.eps, s.fr, dv0, dv1, dv2, ds1, ds2, dt);
    if (g.dL_dtriangles) {
#pragma unroll
        for (int k = 0; k < 9; k++) g.dL_dtriangles[9 * (size_t)f + k] = dt[k];
    }
    if (g.dL_dvertices && !a.triangles_in) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            GMS_ATOMIC_ADD(&g.dL_dvertices[3 * s.vi[c]], dt[3 * c]);
            GMS_ATOMIC_ADD(&g.dL_dvertices[3 * s.vi[c] + 1], dt[3 * c + 1]);
            GMS_ATOMIC_ADD(&g.dL_dvertices[3 * s.vi[c] + 2], dt[3 * c + 2]);
        }
    }
}

template <int ACT>
GMS_HD void gms_expand_face_bwd_act(const gms_expand_args& a, const gms_expand_grads& g, int f, int fl) {
    GmsFaceState s;
    gms_expand_face_load(a, f, s);
    gms_expand_face_frame(a, s);
    float dt[9];
#pragma unroll
    for (int k = 0; k < 9; k++) dt[k] = 0.f;
    float dq[4] = {0.f, 0.f, 0.f, 0.f};
    float ds1 = 0.f, ds2 = 0.f;
    for (int k = 0; k < a.K; k++) gms_expand_splat_bwd<ACT>(a, g, s, (size_t)fl * a.K + k, dt, dq, ds1, ds2);
    gms_expand_face_bwd_tail(a, g, s, f, dt, dq, ds1, ds2);
}

// Whole face with the activation the arguments select (the host shim's entry points; the per-thread kernels call the
// templates above directly).
GMS_HD void gms_expand_face_fwd(const gms_expand_args& a, int f, int fl) {
    if (a.alpha_activation == GMS_ALPHA_SOFTMAX) gms_expand_face_fwd_act<GMS_ALPHA_SOFTMAX>(a, f, fl);
    else gms_expand_face_fwd_act<GMS_ALPHA_RELU>(a, f, fl);
}

GMS_HD void gms_expand_face_bwd(const gms_expand_args& a, const gms_expand_grads& g, int f, int fl) {
    if (a.alpha_activation == GMS_ALPHA_SOFTMAX) gms_expand_face_bwd_act<GMS_ALPHA_SOFTMAX>(a, g, f, fl);
    else gms_expand_face_bwd_act<GMS_ALPHA_RELU>(a, g, f, fl);
}


// ---- gs_points pseudo-mesh path (SURVEY.md section 8f rank 3): every Gaussian carries its own triangle (v1, v2, v3);
// PointsGaussianModel.prepare_scaling_rot  games/flat_splatting/scene/points_gaussian_model.py:61-104 and the per-frame
// call in renderer/gaussian_points_animated_renderer/__init__.py:61-66 (_xyz = triangles[:, 0]).  Forward only: the
// reference uses it under torch.no_grad() in scripts/render_points_time_animated.py.
// The core takes the triangle's three vertices from wherever the caller holds them (the triangles array, or registers of
// the mesh-driven kernel); `i` indexes the outputs.
GMS_HD void gms_points_core_fwd(const gms_points_args& a, int i, const float* v1, const float* v2, const float* v3) {
    float e2[3], e3[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { e2[k] = v2[k] - v1[k]; e3[k] = v3[k] - v1[k]; }
    GmsFrame f;                                   // v0 <- r1 (normal), v1 <- r2, v2 <- r3: rotation COLUMNS
    f.n[0] = e2[1] * e3[2] - e2[2] * e3[1];
    f.n[1] = e2[2] * e3[0] - e2[0] * e3[2];
    f.n[2] = e2[0] * e3[1] - e2[1] * e3[0];
    f.nn = gms_norm3(f.n);
    const float s2 = gms_norm3(e2) + a.eps;
    const float inn = 1.0f / (f.nn + a.eps);
#pragma unroll
    for (int k = 0; k < 3; k++) { f.v0[k] = f.n[k] * inn; f.v1[k] = e2[k] / s2; }
    const float d0 = gms_dotv(e3, f.v0), d1 = gms_dotv(e3, f.v1);
    float u[3];
#pragma unroll
    for (int k = 0; k < 3; k++) u[k] = e3[k] - d0 * f.v0[k] - d1 * f.v1[k];
    const float lu = gms_norm3(u) + a.eps;
#pragma unroll
    for (int k = 0; k < 3; k++) f.v2[k] = u[k] / lu;
    const float s3 = gms_dotv(e3, f.v2);
    float q[4];
    GmsQuatAux ax;
    gms_frame_quat(f, q, ax);
    if (a.xyz) { a.xyz[3 * (size_t)i] = v1[0]; a.xyz[3 * (size_t)i + 1] = v1[1]; a.xyz[3 * (size_t)i + 2] = v1[2]; }
    if (a.scaling_log) { a.scaling_log[2 * (size_t)i] = logf(fabsf(s2)); a.scaling_log[2 * (size_t)i + 1] = logf(fabsf(s3)); }
    if (a.scaling_act) {      // get_scaling = cat([eps], exp(_scaling))  (points_gaussian_model.py:106-109)
        a.scaling_act[3 * (size_t)i] = a.eps;
        a.scaling_act[3 * (size_t)i + 1] = expf(logf(fabsf(s2)));
        a.scaling_act[3 * (size_t)i + 2] = expf(logf(fabsf(s3)));
    }
    if (a.rotation_raw) { float* o = a.rotation_raw + 4 * (size_t)i; o[0] = q[0]; o[1] = q[1]; o[2] = q[2]; o[3] = q[3]; }
    if (a.rotation_act) {
        const float qn = fmaxf(GMS_SQRTN(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
        float* o = a.rotation_act + 4 * (size_t)i; o[0] = GMS_DIVN(q[0], qn); o[1] = GMS_DIVN(q[1], qn); o[2] = GMS_DIVN(q[2], qn); o[3] = GMS_DIVN(q[3], qn);
    }
}

GMS_HD void gms_points_face_fwd(const gms_points_args& a, int i) {
    const float* t = a.triangles + 9 * (size_t)i;
    gms_points_core_fwd(a, i, t, t + 3, t + 6);
}

// ---- mesh-driven pseudo-mesh: every pseudo-triangle is bound to the nearest face of a driving mesh and follows it
// (scripts/edit_pseudomesh_based_on_estimated_mesh.py:8-82).  Every operation is an explicit round-to-nearest one with no
// contraction, so numpy (float32 / float64) restates each function bit for bit (tests/pseudomesh_oracle.py).
#if defined(__CUDA_ARCH__)
#define GMS_DMUL(a, b) __dmul_rn((a), (b))
#define GMS_DADD(a, b) __dadd_rn((a), (b))
#define GMS_DSUB(a, b) __dsub_rn((a), (b))
#define GMS_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define GMS_DMUL(a, b) ((a) * (b))
#define GMS_DADD(a, b) ((a) + (b))
#define GMS_DSUB(a, b) ((a) - (b))
#define GMS_DDIV(a, b) ((a) / (b))
#endif

// A face's frame: the skewed basis (n, e1, e2) of the reference (:32-43, :62-70), n = normalise(cross(v2 - v1, v3 - v1)),
// e1 = normalise(v2 - v1), e2 = normalise(v3 - v1).  IEEE division and square root: the norms may be 0.  Returns true when
// the face is degenerate (one of the three norms is exactly 0; its frame is then non-finite).
struct GmsPmFrame { float n[3], e1[3], e2[3]; };

GMS_HD float gms_pm_norm(const float* v) {
    return GMS_SQRT(GMS_ADD(GMS_ADD(GMS_MUL(v[0], v[0]), GMS_MUL(v[1], v[1])), GMS_MUL(v[2], v[2])));
}

GMS_HD bool gms_pm_frame(const float* v1, const float* v2, const float* v3, GmsPmFrame& f) {
    float a[3], b[3], c[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { a[k] = GMS_SUB(v2[k], v1[k]); b[k] = GMS_SUB(v3[k], v1[k]); }
    c[0] = GMS_SUB(GMS_MUL(a[1], b[2]), GMS_MUL(a[2], b[1]));
    c[1] = GMS_SUB(GMS_MUL(a[2], b[0]), GMS_MUL(a[0], b[2]));
    c[2] = GMS_SUB(GMS_MUL(a[0], b[1]), GMS_MUL(a[1], b[0]));
    const float la = gms_pm_norm(a), lb = gms_pm_norm(b), lc = gms_pm_norm(c);
#pragma unroll
    for (int k = 0; k < 3; k++) { f.n[k] = GMS_DIV(c[k], lc); f.e1[k] = GMS_DIV(a[k], la); f.e2[k] = GMS_DIV(b[k], lb); }
    return la == 0.f || lb == 0.f || lc == 0.f;
}

// Centroid of a pseudo-triangle or a face, ((v0 + v1) + v2) / 3.
GMS_HD void gms_pm_centroid(const float* v0, const float* v1, const float* v2, float* m) {
#pragma unroll
    for (int k = 0; k < 3; k++) m[k] = GMS_DIV(GMS_ADD(GMS_ADD(v0[k], v1[k]), v2[k]), 3.0f);
}

// Squared distance between two centroids in double, as sklearn's Euclidean rdist sums it: (dx*dx + dy*dy) + dz*dz.
GMS_HD double gms_pm_dist2(double qx, double qy, double qz, double cx, double cy, double cz) {
    const double dx = GMS_DSUB(qx, cx), dy = GMS_DSUB(qy, cy), dz = GMS_DSUB(qz, cz);
    return GMS_DADD(GMS_DADD(GMS_DMUL(dx, dx), GMS_DMUL(dy, dy)), GMS_DMUL(dz, dz));
}

GMS_HD void gms_pm_dcross(const double* a, const double* b, double* c) {
    c[0] = GMS_DSUB(GMS_DMUL(a[1], b[2]), GMS_DMUL(a[2], b[1]));
    c[1] = GMS_DSUB(GMS_DMUL(a[2], b[0]), GMS_DMUL(a[0], b[2]));
    c[2] = GMS_DSUB(GMS_DMUL(a[0], b[1]), GMS_DMUL(a[1], b[0]));
}

GMS_HD double gms_pm_ddot(const double* a, const double* b) {
    return GMS_DADD(GMS_DADD(GMS_DMUL(a[0], b[0]), GMS_DMUL(a[1], b[1])), GMS_DMUL(a[2], b[2]));
}

// Coefficients of the three pseudo-vertices w_j in the face's frame: [n|e1|e2] c_j = w_j - v1 (the reference's
// torch.linalg.solve, :52-54), solved in double through the adjugate and rounded to fp32.  c[3*j + k] multiplies n, e1, e2
// for k = 0, 1, 2.
GMS_HD void gms_pm_coeffs(const GmsPmFrame& f, const float* v1, const float* w, float* c) {
    double n[3], e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { n[k] = f.n[k]; e1[k] = f.e1[k]; e2[k] = f.e2[k]; }
    double r0[3], r1[3], r2[3];           // rows of det * inverse
    gms_pm_dcross(e1, e2, r0);
    gms_pm_dcross(e2, n, r1);
    gms_pm_dcross(n, e1, r2);
    const double det = gms_pm_ddot(n, r0);
#pragma unroll
    for (int j = 0; j < 3; j++) {
        double d[3];
#pragma unroll
        for (int k = 0; k < 3; k++) d[k] = GMS_DSUB((double)w[3 * j + k], (double)v1[k]);
        c[3 * j] = (float)GMS_DDIV(gms_pm_ddot(d, r0), det);
        c[3 * j + 1] = (float)GMS_DDIV(gms_pm_ddot(d, r1), det);
        c[3 * j + 2] = (float)GMS_DDIV(gms_pm_ddot(d, r2), det);
    }
}

// Re-pose: w_j = ((v1 + c_j0 n) + c_j1 e1) + c_j2 e2 in the (driving) face's frame (calc_new_vertices_position, :8-12).
GMS_HD void gms_pm_repose(const GmsPmFrame& f, const float* v1, const float* c, float* w) {
#pragma unroll
    for (int j = 0; j < 3; j++) {
#pragma unroll
        for (int k = 0; k < 3; k++)
            w[3 * j + k] = GMS_ADD(GMS_ADD(GMS_ADD(v1[k], GMS_MUL(c[3 * j], f.n[k])), GMS_MUL(c[3 * j + 1], f.e1[k])),
                                   GMS_MUL(c[3 * j + 2], f.e2[k]));
    }
}

// PointsGaussianModel.prepare_vertices (games/flat_splatting/scene/points_gaussian_model.py:28-59): pseudo-mesh triangle of
// one flat Gaussian.  scales = (eps, exp(_scaling[-2]), exp(_scaling[-1])) (:106-109); R = build_rotation(_rotation)
// (utils/general_utils.py:158-179, normalises q); arms along R's 2nd and 3rd COLUMNS (R.transpose(-2,-1)[:, 1|2]);
// the longer arm becomes v2 (mask = s_2 > s_3, :43-52).
GMS_HD void gms_points_vertices_fwd(const gms_points_vertices_args& a, int i) {
    const float* c = a.xyz + 3 * (size_t)i;
    const float* sl = a.scaling_log + (size_t)a.scaling_cols * i + (a.scaling_cols - 2);
    const float* qr = a.rotation_raw + 4 * (size_t)i;
    const float s2 = expf(sl[0]), s3 = expf(sl[1]);
    const float nrm = sqrtf(qr[0] * qr[0] + qr[1] * qr[1] + qr[2] * qr[2] + qr[3] * qr[3]);
    const float r = qr[0] / nrm, x = qr[1] / nrm, y = qr[2] / nrm, z = qr[3] / nrm;
    const float ax2[3] = {2.0f * (x * y - r * z), 1.0f - 2.0f * (x * x + z * z), 2.0f * (y * z + r * x)};
    const float ax3[3] = {2.0f * (x * z + r * y), 2.0f * (y * z - r * x), 1.0f - 2.0f * (x * x + y * y)};
    float p2[3], p3[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { p2[k] = c[k] + s2 * ax2[k]; p3[k] = c[k] + s3 * ax3[k]; }
    const bool keep = s2 > s3;
    float* t = a.triangles + 9 * (size_t)i;
#pragma unroll
    for (int k = 0; k < 3; k++) { t[k] = c[k]; t[3 + k] = keep ? p2[k] : p3[k]; t[6 + k] = keep ? p3[k] : p2[k]; }
}

#if defined(__CUDACC__)

// ------------------------------------------------------------------------------------------ expansion kernels
// One thread per face.  The forward's per-Gaussian streams (K rows per face: 36-48 B per thread, i.e. a 36-48 B stride
// between lanes) are staged through shared memory: the block copies its contiguous slice of every stream with fully
// coalesced accesses, the per-face maths then reads / writes shared memory (gms_expand_face_* with fl = slot in the block).
// STAGED = false is the direct variant, for K whose staging would exceed 48 KB.  The backward reads and writes its rows
// directly: staging them measured no faster (DESIGN.md 3.7).
constexpr int GMS_EXP_BLOCK = 128;

__device__ __forceinline__ const float* exp_stage_in(const float* src, int width, size_t g0, int ng, int cap, float*& sm) {
    if (!src) return nullptr;
    float* dst = sm; sm += (size_t)cap * width;
    const float* s0 = src + g0 * width;
    for (int i = threadIdx.x; i < ng * width; i += GMS_EXP_BLOCK) dst[i] = s0[i];
    return dst;
}
__device__ __forceinline__ float* exp_stage_out(float* dst, int width, int cap, float*& sm) {
    if (!dst) return nullptr;
    float* b = sm; sm += (size_t)cap * width;
    return b;
}
__device__ __forceinline__ void exp_stage_flush(float* dst, const float* buf, int width, size_t g0, int ng) {
    if (!dst) return;
    float* d0 = dst + g0 * width;
    for (int i = threadIdx.x; i < ng * width; i += GMS_EXP_BLOCK) d0[i] = buf[i];
}

template <bool STAGED, int ACT>
__global__ void __launch_bounds__(GMS_EXP_BLOCK) k_expand_fwd(gms_expand_args a) {
    const int f0 = blockIdx.x * GMS_EXP_BLOCK, f = f0 + threadIdx.x;
    if (!STAGED) {
        if (f < a.F) gms_expand_face_fwd_act<ACT>(a, f, f);
        return;
    }
    extern __shared__ float4 exp_smem4[];
    float* sm = reinterpret_cast<float*>(exp_smem4);
    const int nf = min(GMS_EXP_BLOCK, a.F - f0), ng = nf * a.K, cap = GMS_EXP_BLOCK * a.K;
    const size_t g0 = (size_t)f0 * a.K;
    gms_expand_args l = a;
    l.alpha_raw = exp_stage_in(a.alpha_raw, 3, g0, ng, cap, sm);
    l.scale_raw = exp_stage_in(a.scale_raw, 1, g0, ng, cap, sm);
    l.alpha = exp_stage_out(a.alpha, 3, cap, sm);
    l.xyz = exp_stage_out(a.xyz, 3, cap, sm);
    l.scaling_log = exp_stage_out(a.scaling_log, 3, cap, sm);
    l.scaling_act = exp_stage_out(a.scaling_act, 3, cap, sm);
    l.rotation_raw = exp_stage_out(a.rotation_raw, 4, cap, sm);
    l.rotation_act = exp_stage_out(a.rotation_act, 4, cap, sm);
    __syncthreads();
    if (f < a.F) gms_expand_face_fwd_act<ACT>(l, f, threadIdx.x);
    __syncthreads();
    exp_stage_flush(a.alpha, l.alpha, 3, g0, ng);
    exp_stage_flush(a.xyz, l.xyz, 3, g0, ng);
    exp_stage_flush(a.scaling_log, l.scaling_log, 3, g0, ng);
    exp_stage_flush(a.scaling_act, l.scaling_act, 3, g0, ng);
    exp_stage_flush(a.rotation_raw, l.rotation_raw, 4, g0, ng);
    exp_stage_flush(a.rotation_act, l.rotation_act, 4, g0, ng);
}

template <int ACT>
__global__ void __launch_bounds__(GMS_EXP_BLOCK) k_expand_bwd(gms_expand_args a, gms_expand_grads g) {
    const int f = blockIdx.x * GMS_EXP_BLOCK + threadIdx.x;
    if (f < a.F) gms_expand_face_bwd_act<ACT>(a, g, f, f);
}

// Splat-parallel expansion for many splats per face (gs_flame: K = 100 on ~10k faces).  One warp per face: every lane reads
// the face and evaluates its frame and quaternion in lockstep (one instruction stream per face, as cheap as one lane
// computing them and broadcasting the result, without the shuffles), then lane j handles splats j, j + 32, ...: consecutive
// lanes touch consecutive rows, so every per-Gaussian stream is read and written coalesced without staging.  Each splat is
// the per-thread kernel's gms_expand_splat_* call, so the forward is bit-identical to it.  The backward sums each lane's
// dt / dq / ds1 / ds2 partials over its splats, reduces them across the warp (butterfly), and lane 0 finishes the face: one
// set of vertex atomics per face, as in the per-thread kernel.  Only the order of the sum over K differs.
// Softmax weights only: relu weights (gs_mesh) always run the per-thread kernels.
constexpr int GMS_EXP_WIDE_BLOCK = 128;                     // 4 faces per block
constexpr int GMS_EXP_WIDE_MIN_K = 16;                      // softmax weights with K >= this run these kernels (DESIGN.md 4.5)

__global__ void __launch_bounds__(GMS_EXP_WIDE_BLOCK) k_expand_wide_fwd(gms_expand_args a) {
    const int f = blockIdx.x * (GMS_EXP_WIDE_BLOCK / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= a.F) return;
    GmsFaceState s;
    gms_expand_face_load(a, f, s);
    if (a.triangles && lane == 0) {
#pragma unroll
        for (int k = 0; k < 9; k++) a.triangles[9 * (size_t)f + k] = s.t[k];
    }
    gms_expand_face_frame(a, s);
    for (int k = lane; k < a.K; k += 32) gms_expand_splat_fwd<GMS_ALPHA_SOFTMAX>(a, s, (size_t)f * a.K + k);
}

__global__ void __launch_bounds__(GMS_EXP_WIDE_BLOCK) k_expand_wide_bwd(gms_expand_args a, gms_expand_grads g) {
    const int f = blockIdx.x * (GMS_EXP_WIDE_BLOCK / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= a.F) return;                                   // whole warps: f is uniform across the warp
    GmsFaceState s;
    gms_expand_face_load(a, f, s);
    gms_expand_face_frame(a, s);
    float acc[15];                                          // dt[9], dq[4], ds1, ds2
#pragma unroll
    for (int i = 0; i < 15; i++) acc[i] = 0.f;
    for (int k = lane; k < a.K; k += 32)
        gms_expand_splat_bwd<GMS_ALPHA_SOFTMAX>(a, g, s, (size_t)f * a.K + k, acc, acc + 9, acc[13], acc[14]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int i = 0; i < 15; i++) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
    }
    if (lane == 0) gms_expand_face_bwd_tail(a, g, s, f, acc, acc + 9, acc[13], acc[14]);
}

__global__ void __launch_bounds__(128) k_points_expand_fwd(gms_points_args a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    gms_points_face_fwd(a, i);
}

__global__ void __launch_bounds__(128) k_points_vertices(gms_points_vertices_args a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    gms_points_vertices_fwd(a, i);
}

// ------------------------------------------------------------------------------------------ mesh-driven pseudo-mesh
// scripts/edit_pseudomesh_based_on_estimated_mesh.py:14-94: bind every pseudo-triangle to the nearest face of a driving mesh
// (nearest centroid, brute force), then re-pose it from any pose of that mesh (gms_expand.cuh: gms_pm_*).
#define GMS_PM_BLOCK 128
#define GMS_PM_TILE 512        // face centroids staged through shared memory per pass

__device__ __forceinline__ void pm_load_face(const float* __restrict__ vertices, const int64_t* __restrict__ faces, int f, float* v) {
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const int64_t vi = faces[3 * (size_t)f + c];
        v[3 * c] = vertices[3 * vi]; v[3 * c + 1] = vertices[3 * vi + 1]; v[3 * c + 2] = vertices[3 * vi + 2];
    }
}

// Per face: (centroid, 1 if degenerate else 0), and the number of degenerate faces.
__global__ void __launch_bounds__(GMS_PM_BLOCK) k_pseudomesh_faces(int F, const float* __restrict__ vertices,
                                                                    const int64_t* __restrict__ faces, float4* __restrict__ cent,
                                                                    uint32_t* __restrict__ n_degenerate) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    float v[9], m[3];
    pm_load_face(vertices, faces, f, v);
    GmsPmFrame fr;
    const bool deg = gms_pm_frame(v, v + 3, v + 6, fr);
    gms_pm_centroid(v, v + 3, v + 6, m);
    cent[f] = make_float4(m[0], m[1], m[2], deg ? 1.f : 0.f);
    if (deg) atomicAdd(n_degenerate, 1u);
}

// One thread per pseudo-triangle: nearest non-degenerate face centroid (double distance, lowest index on a tie; the first
// non-degenerate face is taken whatever its distance, so a non-finite query still binds in range), then the 9 coefficients.
__global__ void __launch_bounds__(GMS_PM_BLOCK) k_pseudomesh_bind(int P, int F, const float* __restrict__ triangles,
                                                                   const float* __restrict__ vertices, const int64_t* __restrict__ faces,
                                                                   const float4* __restrict__ cent, int32_t* __restrict__ face_out,
                                                                   float* __restrict__ coeffs) {
    __shared__ double sx[GMS_PM_TILE], sy[GMS_PM_TILE], sz[GMS_PM_TILE];
    __shared__ uint8_t sdeg[GMS_PM_TILE];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float w[9], q[3] = {0.f, 0.f, 0.f};
    if (i < P) {
#pragma unroll
        for (int k = 0; k < 9; k++) w[k] = triangles[9 * (size_t)i + k];
        gms_pm_centroid(w, w + 3, w + 6, q);
    }
    const double qx = q[0], qy = q[1], qz = q[2];
    double best = 0.0;
    int bi = -1;
    for (int t0 = 0; t0 < F; t0 += GMS_PM_TILE) {
        const int n = min(GMS_PM_TILE, F - t0);
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const float4 c = cent[t0 + j];
            sx[j] = c.x; sy[j] = c.y; sz[j] = c.z; sdeg[j] = c.w != 0.f;
        }
        __syncthreads();
        for (int j = 0; j < n; j++) {
            if (sdeg[j]) continue;
            const double d = gms_pm_dist2(qx, qy, qz, sx[j], sy[j], sz[j]);
            if (d < best || bi < 0) { best = d; bi = t0 + j; }
        }
    }
    if (i >= P) return;
    float v[9], c[9];
    pm_load_face(vertices, faces, bi, v);
    GmsPmFrame fr;
    gms_pm_frame(v, v + 3, v + 6, fr);
    gms_pm_coeffs(fr, v, w, c);
    face_out[i] = bi;
#pragma unroll
    for (int k = 0; k < 9; k++) coeffs[9 * (size_t)i + k] = c[k];
}

// The pseudo-triangle of binding i in the driving pose (vertices, faces).
__device__ __forceinline__ void pm_reposed(const gms_pseudomesh_repose_args& a, int i, float* w) {
    float v[9], c[9];
    pm_load_face(a.vertices, a.faces, a.face[i], v);
#pragma unroll
    for (int k = 0; k < 9; k++) c[k] = a.coeffs[9 * (size_t)i + k];
    GmsPmFrame fr;
    gms_pm_frame(v, v + 3, v + 6, fr);
    gms_pm_repose(fr, v, c, w);
}

__global__ void __launch_bounds__(GMS_PM_BLOCK) k_pseudomesh_repose(gms_pseudomesh_repose_args a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    float w[9];
    pm_reposed(a, i, w);
#pragma unroll
    for (int k = 0; k < 9; k++) a.triangles[9 * (size_t)i + k] = w[k];
}

// Re-pose + the gs_points expansion in one pass (the triangles never reach global memory).  The core reads the re-posed
// triangle from a per-thread slot in shared memory, as k_points_expand_fwd reads it from the triangles array: the core's
// fp32 expressions leave contraction to the compiler, and reading the vertices from memory in both kernels keeps its
// choices, and so the Gaussians, bit-identical to the triangles path.  A Gaussian whose re-posed triangle is not finite (its
// driving face is degenerate in this pose) is placed at the camera centre, -R^T t of the view matrix: its view-space depth
// is ~0 <= the near plane, so the preprocess's first test culls it (radius 0, no tile) before it reads anything else of it.
__global__ void __launch_bounds__(GMS_PM_BLOCK) k_points_bound_expand_fwd(gms_pseudomesh_repose_args r, gms_points_args a,
                                                                           const float* __restrict__ view) {
    __shared__ float tri[GMS_PM_BLOCK * 9];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.P) return;
    float w[9];
    pm_reposed(r, i, w);
    float* t = tri + 9 * threadIdx.x;
#pragma unroll
    for (int k = 0; k < 9; k++) t[k] = w[k];
    asm volatile("" ::: "memory");      // no store-to-load forwarding: the core loads its vertices, as in the triangles path
    gms_points_core_fwd(a, i, t, t + 3, t + 6);
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 9; k++) finite = finite && isfinite(w[k]);
    if (!finite) {
#pragma unroll
        for (int j = 0; j < 3; j++)
            a.xyz[3 * (size_t)i + j] = -(view[4 * j] * view[12] + view[4 * j + 1] * view[13] + view[4 * j + 2] * view[14]);
    }
}

#endif  // __CUDACC__
