// gms_preprocess.cuh -- per-Gaussian maths of the preprocess stage, forward and backward.
// Host+device: the CUDA kernels in gms_kernels.cu call these per thread; tests/hostshim compiles the
// same functions with g++ to unit-test them against the oracle without a GPU.
//
// Replaces [upstream forward.cu: preprocessCUDA, computeCov3D, computeCov2D, computeColorFromSH] and
// [upstream backward.cu: computeCov2DCUDA, preprocessCUDA, computeCov3D, computeColorFromSH] of
// graphdeco-inria/diff-gaussian-rasterization (reference call site renderer/gaussian_renderer/__init__.py:94-102).
// Python restatements the reference ships and that pin these maths: utils/sh_utils.py:57-112 (SH),
// utils/general_utils.py:144-190 (cov3D), utils/graphics_utils.py:22-29 (homogeneous divide).
#pragma once
#include "gms_common.cuh"

// rotation matrix (row-major) of an un-normalised quaternion (r,x,y,z); utils/general_utils.py:170-178
GMS_HD void gms_quat_to_R(const float* q, float* R) {
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = GMS_SUB(1.f, GMS_MUL(2.f, GMS_FMA(y, y, GMS_MUL(z, z))));
    R[1] = GMS_MUL(2.f, GMS_FMA(x, y, -GMS_MUL(r, z)));
    R[2] = GMS_MUL(2.f, GMS_FMA(x, z, GMS_MUL(r, y)));
    R[3] = GMS_MUL(2.f, GMS_FMA(x, y, GMS_MUL(r, z)));
    R[4] = GMS_SUB(1.f, GMS_MUL(2.f, GMS_FMA(x, x, GMS_MUL(z, z))));
    R[5] = GMS_MUL(2.f, GMS_FMA(y, z, -GMS_MUL(r, x)));
    R[6] = GMS_MUL(2.f, GMS_FMA(x, z, -GMS_MUL(r, y)));
    R[7] = GMS_MUL(2.f, GMS_FMA(y, z, GMS_MUL(r, x)));
    R[8] = GMS_SUB(1.f, GMS_MUL(2.f, GMS_FMA(x, x, GMS_MUL(y, y))));
}

// Sigma = (R S)(R S)^T packed [00,01,02,11,12,22]
GMS_HD void gms_cov3d(const float* scale, float mod, const float* q, float* cov6) {
    float R[9], M[9];
    gms_quat_to_R(q, R);
    const float s0 = GMS_MUL(mod, scale[0]), s1 = GMS_MUL(mod, scale[1]), s2 = GMS_MUL(mod, scale[2]);
#pragma unroll
    for (int i = 0; i < 3; i++) {
        M[3 * i + 0] = GMS_MUL(R[3 * i + 0], s0);
        M[3 * i + 1] = GMS_MUL(R[3 * i + 1], s1);
        M[3 * i + 2] = GMS_MUL(R[3 * i + 2], s2);
    }
    cov6[0] = gms_dot3(M[0], M[0], M[1], M[1], M[2], M[2]);
    cov6[1] = gms_dot3(M[0], M[3], M[1], M[4], M[2], M[5]);
    cov6[2] = gms_dot3(M[0], M[6], M[1], M[7], M[2], M[8]);
    cov6[3] = gms_dot3(M[3], M[3], M[4], M[4], M[5], M[5]);
    cov6[4] = gms_dot3(M[3], M[6], M[4], M[7], M[5], M[8]);
    cov6[5] = gms_dot3(M[6], M[6], M[7], M[7], M[8], M[8]);
}

struct GmsCov2D {
    float M0[3], M1[3];  // rows of J*W
    float tx, ty, tz;    // clamped view-space point
    float xmul, ymul;    // 0 where the guard-band clamp was active
    float a, b, c;       // raw (undilated) 2D covariance
};

// EWA projection, Appendix A.1 step 4
GMS_HD void gms_cov2d(const float* pview, const float* cov6, const float* view, float focal_x, float focal_y,
                      float tanfovx, float tanfovy, GmsCov2D& o) {
    const float tz = pview[2];
    const float limx = GMS_MUL(1.3f, tanfovx), limy = GMS_MUL(1.3f, tanfovy);
    const float txtz = GMS_DIVP(pview[0], tz), tytz = GMS_DIVP(pview[1], tz);
    o.xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    o.ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    const float tx = GMS_MUL(fminf(limx, fmaxf(-limx, txtz)), tz);
    const float ty = GMS_MUL(fminf(limy, fmaxf(-limy, tytz)), tz);
    o.tx = tx; o.ty = ty; o.tz = tz;
    const float tz2 = GMS_MUL(tz, tz);
    const float J00 = GMS_DIVP(focal_x, tz);
    const float J02 = GMS_DIVP(-GMS_MUL(focal_x, tx), tz2);
    const float J11 = GMS_DIVP(focal_y, tz);
    const float J12 = GMS_DIVP(-GMS_MUL(focal_y, ty), tz2);
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const float W0j = view[4 * j + 0], W1j = view[4 * j + 1], W2j = view[4 * j + 2];
        o.M0[j] = GMS_FMA(J02, W2j, GMS_MUL(J00, W0j));
        o.M1[j] = GMS_FMA(J12, W2j, GMS_MUL(J11, W1j));
    }
    const float S00 = cov6[0], S01 = cov6[1], S02 = cov6[2], S11 = cov6[3], S12 = cov6[4], S22 = cov6[5];
    const float v0 = gms_dot3(S00, o.M0[0], S01, o.M0[1], S02, o.M0[2]);
    const float v1 = gms_dot3(S01, o.M0[0], S11, o.M0[1], S12, o.M0[2]);
    const float v2 = gms_dot3(S02, o.M0[0], S12, o.M0[1], S22, o.M0[2]);
    const float w0 = gms_dot3(S00, o.M1[0], S01, o.M1[1], S02, o.M1[2]);
    const float w1 = gms_dot3(S01, o.M1[0], S11, o.M1[1], S12, o.M1[2]);
    const float w2 = gms_dot3(S02, o.M1[0], S12, o.M1[1], S22, o.M1[2]);
    o.a = gms_dot3(o.M0[0], v0, o.M0[1], v1, o.M0[2], v2);
    o.b = gms_dot3(o.M1[0], v0, o.M1[1], v1, o.M1[2], v2);
    o.c = gms_dot3(o.M1[0], w0, o.M1[1], w1, o.M1[2], w2);
}

// SH basis (utils/sh_utils.py:74-100); B must hold 16 floats
GMS_HD void gms_sh_basis(int deg, float x, float y, float z, float* B) {
    B[0] = GMS_SH_C0;
    if (deg > 0) {
        B[1] = -GMS_SH_C1 * y; B[2] = GMS_SH_C1 * z; B[3] = -GMS_SH_C1 * x;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            B[4] = GMS_SH_C2_0 * xy; B[5] = GMS_SH_C2_1 * yz;
            B[6] = GMS_SH_C2_2 * (2.0f * zz - xx - yy);
            B[7] = GMS_SH_C2_3 * xz; B[8] = GMS_SH_C2_4 * (xx - yy);
            if (deg > 2) {
                B[9] = GMS_SH_C3_0 * y * (3.0f * xx - yy);
                B[10] = GMS_SH_C3_1 * xy * z;
                B[11] = GMS_SH_C3_2 * y * (4.0f * zz - xx - yy);
                B[12] = GMS_SH_C3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
                B[13] = GMS_SH_C3_4 * x * (4.0f * zz - xx - yy);
                B[14] = GMS_SH_C3_5 * z * (xx - yy);
                B[15] = GMS_SH_C3_6 * x * (xx - 3.0f * yy);
            }
        }
    }
}

struct GmsPre {           // everything preprocess produces for one Gaussian
    int radius;
    float px, py, depth;
    float cov6[6];
    float conx, cony, conz, opac;
    int x0, y0, x1, y1;
    uint32_t tiles;
};

// Geometry part of preprocess (steps 1-8, 10 of Appendix A.1).  Returns false when culled.
// `cov6_in` non-NULL => precomputed covariance; else scale/rot are used.
GMS_HD bool gms_preprocess_geom(const float* mean, const float* scale, const float* rot, const float* cov6_in,
                                float opacity, const float* view, const float* proj, int W, int H,
                                float tanfovx, float tanfovy, float focal_x, float focal_y, float mod,
                                int antialiasing, int gx, int gy, GmsPre& o) {
    o.radius = 0; o.tiles = 0;
    float pview[3];
    gms_xform4x3(view, mean[0], mean[1], mean[2], pview);
    if (pview[2] <= GMS_NEAR) return false;
    float phom[4];
    gms_xform4x4(proj, mean[0], mean[1], mean[2], phom);
    const float pw = GMS_DIVP(1.0f, GMS_ADD(phom[3], 0.0000001f));
    const float pprojx = GMS_MUL(phom[0], pw), pprojy = GMS_MUL(phom[1], pw);
    if (cov6_in) {
#pragma unroll
        for (int k = 0; k < 6; k++) o.cov6[k] = cov6_in[k];
    } else {
        gms_cov3d(scale, mod, rot, o.cov6);
    }
    GmsCov2D c2;
    gms_cov2d(pview, o.cov6, view, focal_x, focal_y, tanfovx, tanfovy, c2);
    float a = c2.a, b = c2.b, c = c2.c;
    const float det_cov = GMS_FMA(a, c, -GMS_MUL(b, b));
    a = GMS_ADD(a, GMS_HVAR); c = GMS_ADD(c, GMS_HVAR);
    const float det = GMS_FMA(a, c, -GMS_MUL(b, b));
    if (det == 0.0f) return false;
    float h_scale = 1.0f;
    if (antialiasing) h_scale = GMS_SQRTP(fmaxf(0.000025f, GMS_DIVP(det_cov, det)));
    const float det_inv = GMS_DIVP(1.f, det);
    o.conx = GMS_MUL(c, det_inv); o.cony = GMS_MUL(-b, det_inv); o.conz = GMS_MUL(a, det_inv);
    const float mid = GMS_MUL(0.5f, GMS_ADD(a, c));
    const float disc = GMS_SQRTP(fmaxf(0.1f, GMS_FMA(mid, mid, -det)));
    const float lambda1 = GMS_ADD(mid, disc), lambda2 = GMS_SUB(mid, disc);
    const int my_radius = (int)ceilf(GMS_MUL(3.f, GMS_SQRTP(fmaxf(lambda1, lambda2))));
    o.px = GMS_MUL(GMS_FMA(GMS_ADD(pprojx, 1.0f), (float)W, -1.0f), 0.5f);
    o.py = GMS_MUL(GMS_FMA(GMS_ADD(pprojy, 1.0f), (float)H, -1.0f), 0.5f);
    gms_get_rect(o.px, o.py, my_radius, gx, gy, &o.x0, &o.y0, &o.x1, &o.y1);
    const int area = (o.x1 - o.x0) * (o.y1 - o.y0);
    if (area == 0) return false;
    o.depth = pview[2];
    o.radius = my_radius;
    o.opac = GMS_MUL(opacity, h_scale);
    o.tiles = (uint32_t)area;
    return true;
}

// SH -> RGB (+0.5, clamp at 0, remember the clamp).  sh = [M][3] row of this Gaussian.
GMS_HD void gms_sh_color(int deg, const float* mean, const float* campos, const float* sh, float* rgb,
                         uint8_t* clamped) {
    float dx = mean[0] - campos[0], dy = mean[1] - campos[1], dz = mean[2] - campos[2];
    const float len = GMS_SQRTP(dx * dx + dy * dy + dz * dz);
    dx = GMS_DIVP(dx, len); dy = GMS_DIVP(dy, len); dz = GMS_DIVP(dz, len);
    float B[16];
    gms_sh_basis(deg, dx, dy, dz, B);
    const int nc = (deg + 1) * (deg + 1);
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 16; k++)
            if (k < nc) acc += B[k] * sh[3 * k + ch];
        acc += 0.5f;
        clamped[ch] = acc < 0.f ? 1 : 0;
        rgb[ch] = fmaxf(acc, 0.f);
    }
}

// ------------------------------------------------------------------------------------------ backward
struct GmsPreGradIn {      // per-Gaussian gradients produced by the composite backward
    float dmean2D[2];      // NDC-scaled
    float dconic[3];       // (xx, xy in the stock HALF convention, yy)
    float dopac;           // w.r.t. conic_opacity.w
    float dcolor[3];
    float dinvdepth;
};

struct GmsPreGradOut {
    float dmean3D[3];
    float dcov6[6];
    float dopacity;
    float dscale[3];
    float drot[4];
};

// Appendix A.4 (i),(ii),(iv): everything except the SH part.
GMS_HD void gms_preprocess_backward_geom(const float* mean, const float* scale, const float* rot, const float* cov6,
                                         float opacity_in, const float* view, const float* proj,
                                         float tanfovx, float tanfovy, float focal_x, float focal_y, float mod,
                                         int antialiasing, const GmsPreGradIn& gi, GmsPreGradOut& go) {
    float pview[3];
    gms_xform4x3(view, mean[0], mean[1], mean[2], pview);
    GmsCov2D c2;
    gms_cov2d(pview, cov6, view, focal_x, focal_y, tanfovx, tanfovy, c2);
    const float a0 = c2.a, b = c2.b, c0 = c2.c;
    const float a = a0 + GMS_HVAR, c = c0 + GMS_HVAR;
    const float det_cov = a0 * c0 - b * b;
    const float det = a * c - b * b;
    float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
    if (antialiasing) {
        const float ratio = GMS_DIVP(det_cov, det);
        const float h_scale = GMS_SQRTP(fmaxf(0.000025f, ratio));
        go.dopacity = gi.dopac * h_scale;
        if (ratio > 0.000025f) {
            const float dL_dratio = GMS_DIVP(gi.dopac * opacity_in, 2.f * h_scale);
            const float inv_det = GMS_DIVP(1.f, det);
            const float k = dL_dratio * inv_det * inv_det;
            dL_da += k * (c0 * det - det_cov * c);
            dL_dc += k * (a0 * det - det_cov * a);
            dL_db += k * (-2.f * b * det + 2.f * b * det_cov);
        }
    } else {
        go.dopacity = gi.dopac;
    }
    const float dcx = gi.dconic[0], dcy = gi.dconic[1], dcz = gi.dconic[2];
    const float denom = det;
    // det^2 overflows to +inf for footprints beyond ~6e4 px; IEEE 1/inf = 0 then skips the conic term below.  The branch-free
    // reciprocal is exact only for normal divisors (it gives NaN for inf), so the overflow is taken out by the select.
    const float denom2 = (denom * denom) + 0.0000001f;
    const float denom2inv = denom2 <= 3.402823466e+38f ? GMS_DIVP(1.0f, denom2) : 0.f;
    if (denom2inv != 0.f) {
        dL_da += denom2inv * (-c * c * dcx + 2.f * b * c * dcy + (denom - a * c) * dcz);
        dL_dc += denom2inv * (-a * a * dcz + 2.f * a * b * dcy + (denom - a * c) * dcx);
        dL_db += denom2inv * 2.f * (b * c * dcx - (denom + 2.f * b * b) * dcy + a * b * dcz);
    }
    const float* M0 = c2.M0; const float* M1 = c2.M1;
    float* g6 = go.dcov6;
    g6[0] = M0[0] * M0[0] * dL_da + M0[0] * M1[0] * dL_db + M1[0] * M1[0] * dL_dc;
    g6[3] = M0[1] * M0[1] * dL_da + M0[1] * M1[1] * dL_db + M1[1] * M1[1] * dL_dc;
    g6[5] = M0[2] * M0[2] * dL_da + M0[2] * M1[2] * dL_db + M1[2] * M1[2] * dL_dc;
    g6[1] = 2.f * M0[0] * M0[1] * dL_da + (M0[0] * M1[1] + M0[1] * M1[0]) * dL_db + 2.f * M1[0] * M1[1] * dL_dc;
    g6[2] = 2.f * M0[0] * M0[2] * dL_da + (M0[0] * M1[2] + M0[2] * M1[0]) * dL_db + 2.f * M1[0] * M1[2] * dL_dc;
    g6[4] = 2.f * M0[2] * M0[1] * dL_da + (M0[1] * M1[2] + M0[2] * M1[1]) * dL_db + 2.f * M1[1] * M1[2] * dL_dc;

    // dL/d(J W) = [2 da M0 + db M1 ; 2 dc M1 + db M0] Sigma
    const float S[9] = {cov6[0], cov6[1], cov6[2], cov6[1], cov6[3], cov6[4], cov6[2], cov6[4], cov6[5]};
    float u0[3], u1[3], dM0[3], dM1[3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        u0[j] = 2.f * dL_da * M0[j] + dL_db * M1[j];
        u1[j] = 2.f * dL_dc * M1[j] + dL_db * M0[j];
    }
#pragma unroll
    for (int j = 0; j < 3; j++) {
        dM0[j] = u0[0] * S[j] + u0[1] * S[3 + j] + u0[2] * S[6 + j];
        dM1[j] = u1[0] * S[j] + u1[1] * S[3 + j] + u1[2] * S[6 + j];
    }
    float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const float W0j = view[4 * j + 0], W1j = view[4 * j + 1], W2j = view[4 * j + 2];
        dJ00 += dM0[j] * W0j; dJ02 += dM0[j] * W2j;
        dJ11 += dM1[j] * W1j; dJ12 += dM1[j] * W2j;
    }
    const float tz = GMS_DIVP(1.f, c2.tz), tz2 = tz * tz, tz3 = tz2 * tz;
    const float dL_dtx = c2.xmul * -focal_x * tz2 * dJ02;
    const float dL_dty = c2.ymul * -focal_y * tz2 * dJ12;
    float dL_dtz = -focal_x * tz2 * dJ00 - focal_y * tz2 * dJ11 + (2.f * focal_x * c2.tx) * tz3 * dJ02 +
                   (2.f * focal_y * c2.ty) * tz3 * dJ12;
    dL_dtz -= GMS_DIVP(gi.dinvdepth, pview[2] * pview[2]);
    float dmx = view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
    float dmy = view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
    float dmz = view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;

    float phom[4];
    gms_xform4x4(proj, mean[0], mean[1], mean[2], phom);
    const float m_w = GMS_DIVP(1.0f, phom[3] + 0.0000001f);
    const float mul1 = phom[0] * m_w * m_w, mul2 = phom[1] * m_w * m_w;
    const float g2x = gi.dmean2D[0], g2y = gi.dmean2D[1];
    dmx += (proj[0] * m_w - proj[3] * mul1) * g2x + (proj[1] * m_w - proj[3] * mul2) * g2y;
    dmy += (proj[4] * m_w - proj[7] * mul1) * g2x + (proj[5] * m_w - proj[7] * mul2) * g2y;
    dmz += (proj[8] * m_w - proj[11] * mul1) * g2x + (proj[9] * m_w - proj[11] * mul2) * g2y;
    go.dmean3D[0] = dmx; go.dmean3D[1] = dmy; go.dmean3D[2] = dmz;

    if (scale && rot) {
        float R[9];
        gms_quat_to_R(rot, R);
        const float sv[3] = {mod * scale[0], mod * scale[1], mod * scale[2]};
        float Mx[9];
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
            for (int cc = 0; cc < 3; cc++) Mx[3 * r + cc] = R[3 * r + cc] * sv[cc];
        const float dS[9] = {g6[0], 0.5f * g6[1], 0.5f * g6[2], 0.5f * g6[1], g6[3], 0.5f * g6[4],
                             0.5f * g6[2], 0.5f * g6[4], g6[5]};
        float dR[9];
#pragma unroll
        for (int cc = 0; cc < 3; cc++) {
            float acc = 0.f;
#pragma unroll
            for (int r = 0; r < 3; r++) {
                const float dMx = 2.f * (dS[3 * r] * Mx[cc] + dS[3 * r + 1] * Mx[3 + cc] + dS[3 * r + 2] * Mx[6 + cc]);
                acc += R[3 * r + cc] * dMx;
                dR[3 * r + cc] = dMx * sv[cc];
            }
            go.dscale[cc] = acc * mod;
        }
        const float qr = rot[0], qx = rot[1], qy = rot[2], qz = rot[3];
        go.drot[0] = 2.f * (-qz * dR[1] + qy * dR[2] + qz * dR[3] - qx * dR[5] - qy * dR[6] + qx * dR[7]);
        go.drot[1] = 2.f * (-2.f * qx * (dR[4] + dR[8]) + qy * (dR[1] + dR[3]) + qz * (dR[2] + dR[6]) + qr * (dR[7] - dR[5]));
        go.drot[2] = 2.f * (-2.f * qy * (dR[0] + dR[8]) + qx * (dR[1] + dR[3]) + qr * (dR[2] - dR[6]) + qz * (dR[5] + dR[7]));
        go.drot[3] = 2.f * (-2.f * qz * (dR[0] + dR[4]) + qr * (dR[3] - dR[1]) + qx * (dR[2] + dR[6]) + qy * (dR[5] + dR[7]));
    } else {
        go.dscale[0] = go.dscale[1] = go.dscale[2] = 0.f;
        go.drot[0] = go.drot[1] = go.drot[2] = go.drot[3] = 0.f;
    }
}

// Appendix A.4 (iii): SH backward.  Writes dsh[3*k+ch] for k < (deg+1)^2 (rest zero) and ADDS the view-direction
// term to dmean.  `dsh` may alias `sh` (k_preprocess_bwd's in-place shared-memory row).  dcolor is the (unmasked) colour gradient; clamped masks it.
GMS_HD void gms_sh_backward(int deg, int M, const float* mean, const float* campos, const float* sh,
                            const float* dcolor, const uint8_t* clamped, float* dsh, float* dmean) {
    const float vx = mean[0] - campos[0], vy = mean[1] - campos[1], vz = mean[2] - campos[2];
    const float len = GMS_SQRTP(vx * vx + vy * vy + vz * vz);
    const float x = GMS_DIVP(vx, len), y = GMS_DIVP(vy, len), z = GMS_DIVP(vz, len);
    float g[3];
#pragma unroll
    for (int ch = 0; ch < 3; ch++) g[ch] = clamped[ch] ? 0.f : dcolor[ch];
    float B[16];
    gms_sh_basis(deg, x, y, z, B);
    const int nc = (deg + 1) * (deg + 1);
    // t_k = sum_ch sh[k][ch] * g[ch]   (every read of sh[] precedes the writes of dsh[]: the two may be the same row)
    float t[16];
#pragma unroll
    for (int k = 0; k < 16; k++) t[k] = (k < nc) ? (sh[3 * k] * g[0] + sh[3 * k + 1] * g[1] + sh[3 * k + 2] * g[2]) : 0.f;
#pragma unroll
    for (int k = 0; k < 16; k++) {
        if (dsh && k < M) {     // dsh == NULL: the caller exchanges the masked colour gradient instead (factored SH gradient)
            const float bk = k < nc ? B[k] : 0.f;
            dsh[3 * k + 0] = bk * g[0]; dsh[3 * k + 1] = bk * g[1]; dsh[3 * k + 2] = bk * g[2];
        }
    }
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;
    if (deg > 0) {
        ddy += -GMS_SH_C1 * t[1]; ddz += GMS_SH_C1 * t[2]; ddx += -GMS_SH_C1 * t[3];
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            ddx += GMS_SH_C2_0 * y * t[4];            ddy += GMS_SH_C2_0 * x * t[4];
            ddy += GMS_SH_C2_1 * z * t[5];            ddz += GMS_SH_C2_1 * y * t[5];
            ddx += GMS_SH_C2_2 * (-2.f * x) * t[6];   ddy += GMS_SH_C2_2 * (-2.f * y) * t[6]; ddz += GMS_SH_C2_2 * (4.f * z) * t[6];
            ddx += GMS_SH_C2_3 * z * t[7];            ddz += GMS_SH_C2_3 * x * t[7];
            ddx += GMS_SH_C2_4 * (2.f * x) * t[8];    ddy += GMS_SH_C2_4 * (-2.f * y) * t[8];
            if (deg > 2) {
                ddx += GMS_SH_C3_0 * 6.f * xy * t[9];                ddy += GMS_SH_C3_0 * (3.f * xx - 3.f * yy) * t[9];
                ddx += GMS_SH_C3_1 * yz * t[10];                     ddy += GMS_SH_C3_1 * xz * t[10];  ddz += GMS_SH_C3_1 * xy * t[10];
                ddx += GMS_SH_C3_2 * (-2.f * xy) * t[11];            ddy += GMS_SH_C3_2 * (4.f * zz - xx - 3.f * yy) * t[11]; ddz += GMS_SH_C3_2 * 8.f * yz * t[11];
                ddx += GMS_SH_C3_3 * (-6.f * xz) * t[12];            ddy += GMS_SH_C3_3 * (-6.f * yz) * t[12]; ddz += GMS_SH_C3_3 * (6.f * zz - 3.f * xx - 3.f * yy) * t[12];
                ddx += GMS_SH_C3_4 * (4.f * zz - 3.f * xx - yy) * t[13]; ddy += GMS_SH_C3_4 * (-2.f * xy) * t[13]; ddz += GMS_SH_C3_4 * 8.f * xz * t[13];
                ddx += GMS_SH_C3_5 * 2.f * xz * t[14];               ddy += GMS_SH_C3_5 * (-2.f * yz) * t[14]; ddz += GMS_SH_C3_5 * (xx - yy) * t[14];
                ddx += GMS_SH_C3_6 * (3.f * xx - 3.f * yy) * t[15];  ddy += GMS_SH_C3_6 * (-6.f * xy) * t[15];
            }
        }
    }
    const float dotp = x * ddx + y * ddy + z * ddz;
    dmean[0] += GMS_DIVP(ddx - x * dotp, len);
    dmean[1] += GMS_DIVP(ddy - y * dotp, len);
    dmean[2] += GMS_DIVP(ddz - z * dotp, len);
}
