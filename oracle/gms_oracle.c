/*
 * gms_oracle.c -- CPU ORACLE for the mesh-Gaussian rasterizer hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under gaussian-mesh-splatting_b200/ may
 * include, link or call this file; only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs use it, and only as the
 * checker / the CPU baseline.
 *
 * PARITY STATUS: "parity unpinned" for the rasterizer.  The algorithm lives in
 * the third-party submodule graphdeco-inria/diff-gaussian-rasterization
 * (pinned 59f5f77e3ddbac3ed9db93ec2cfe99ed6c5d121d in /root/reference/.gitmodules:4-6,
 * but the reference's call sites -- renderer/gaussian_renderer/__init__.py:43-57,
 * 94-102 -- need the later antialiasing / inverse-depth API).  Its source is NOT
 * vendored under /root/reference (the directory is empty) and the reference
 * ships no tests or golden vectors for it.  This file restates the published
 * algorithm as specified in SURVEY.md Appendix A.  It is pinned instead against
 *   (1) the pieces the reference DOES ship in Python: SH evaluation
 *       (utils/sh_utils.py:57-112), cov3D = (R S)(R S)^T packing
 *       (utils/general_utils.py:144-190, scene/gaussian_model.py:27-31) and the
 *       projection conventions (utils/graphics_utils.py:22-29,51-71) -- golden
 *       vectors generated from those live under tests/golden/;
 *   (2) an independent dense PyTorch autograd model (oracle/torch_dense.py)
 *       for the compositing forward and every gradient;
 *   (3) closed-form known-answer tests (tests/test_oracle_kat.py).
 *
 * Floating-point convention: every expression that decides an INTEGER output
 * (radii, tile rectangles, depth key bits, hence tiles_touched and the sorted
 * point list) is written as an explicit sequence of IEEE fp32 mul/add/fma/div/
 * sqrt so that the CUDA kernels can replay exactly the same sequence; compile
 * with -ffp-contract=off so gcc adds no fusions of its own.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define GMSO_BLOCK 16
#define GMSO_NCH 3

typedef struct {
    int32_t P;            /* number of Gaussians */
    int32_t D;            /* active SH degree 0..3 */
    int32_t M;            /* SH coefficients stored per Gaussian (16) */
    int32_t W, H;         /* image size */
    float tanfovx, tanfovy;
    float scale_modifier;
    int32_t prefiltered;
    int32_t antialiasing;
    float viewmatrix[16]; /* flat, transposed convention: m[4*c+r] = true (r,c) */
    float projmatrix[16];
    float campos[3];
    float bg[3];
} gmso_settings;

/* SH constants: utils/sh_utils.py:26-43 */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

/* Work statistics of the last composite forward (for DESIGN.md / kernel design, not used by any test):
 * [0] (pixel,splat) pairs visited before the pixel terminated, [1] pairs that blended (alpha >= 1/255),
 * [2] (8x8 quad, splat) pairs with at least one blending pixel, [3] (tile, splat) pairs with >= 1 blending pixel. */
static long long g_stats[4];
void gmso_get_stats(long long* out) { for (int i = 0; i < 4; i++) out[i] = g_stats[i]; }

/* Bounded-sample support for the CPU baseline (bench.py): composite only tiles with tile % stride == 0. */
static int g_tile_stride = 1;
void gmso_set_tile_stride(int s) { g_tile_stride = s > 0 ? s : 1; }

int gmso_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void gmso_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* ---- canonical fp32 sequences (replayed bit-for-bit by the CUDA kernels) ---- */
static inline float dot3_fma(float a0, float b0, float a1, float b1, float a2, float b2) {
    /* ((a0*b0 + a1*b1) + a2*b2) with the two adds fused */
    return fmaf(a2, b2, fmaf(a1, b1, a0 * b0));
}

static inline void xform4x3(const float* m, float x, float y, float z, float* o) {
    o[0] = dot3_fma(m[0], x, m[4], y, m[8], z) + m[12];
    o[1] = dot3_fma(m[1], x, m[5], y, m[9], z) + m[13];
    o[2] = dot3_fma(m[2], x, m[6], y, m[10], z) + m[14];
}

static inline void xform4x4(const float* m, float x, float y, float z, float* o) {
    o[0] = dot3_fma(m[0], x, m[4], y, m[8], z) + m[12];
    o[1] = dot3_fma(m[1], x, m[5], y, m[9], z) + m[13];
    o[2] = dot3_fma(m[2], x, m[6], y, m[10], z) + m[14];
    o[3] = dot3_fma(m[3], x, m[7], y, m[11], z) + m[15];
}

/* rotation matrix of an (unnormalised) quaternion q=(r,x,y,z), row-major;
 * utils/general_utils.py:170-178, Appendix A.1 step 3 */
static inline void quat_to_R(const float* q, float* R) {
    float r = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = 1.f - 2.f * fmaf(y, y, z * z);
    R[1] = 2.f * fmaf(x, y, -(r * z));
    R[2] = 2.f * fmaf(x, z, r * y);
    R[3] = 2.f * fmaf(x, y, r * z);
    R[4] = 1.f - 2.f * fmaf(x, x, z * z);
    R[5] = 2.f * fmaf(y, z, -(r * x));
    R[6] = 2.f * fmaf(x, z, -(r * y));
    R[7] = 2.f * fmaf(y, z, r * x);
    R[8] = 1.f - 2.f * fmaf(x, x, y * y);
}

/* Sigma = (R S)(R S)^T packed [00,01,02,11,12,22]; utils/general_utils.py:144-153 */
static inline void cov3d_from_scale_rot(const float* scale, float mod, const float* q, float* cov6) {
    float R[9], Mx[9];
    quat_to_R(q, R);
    float s0 = mod * scale[0], s1 = mod * scale[1], s2 = mod * scale[2];
    for (int i = 0; i < 3; i++) {
        Mx[3 * i + 0] = R[3 * i + 0] * s0;
        Mx[3 * i + 1] = R[3 * i + 1] * s1;
        Mx[3 * i + 2] = R[3 * i + 2] * s2;
    }
    cov6[0] = dot3_fma(Mx[0], Mx[0], Mx[1], Mx[1], Mx[2], Mx[2]);
    cov6[1] = dot3_fma(Mx[0], Mx[3], Mx[1], Mx[4], Mx[2], Mx[5]);
    cov6[2] = dot3_fma(Mx[0], Mx[6], Mx[1], Mx[7], Mx[2], Mx[8]);
    cov6[3] = dot3_fma(Mx[3], Mx[3], Mx[4], Mx[4], Mx[5], Mx[5]);
    cov6[4] = dot3_fma(Mx[3], Mx[6], Mx[4], Mx[7], Mx[5], Mx[8]);
    cov6[5] = dot3_fma(Mx[6], Mx[6], Mx[7], Mx[7], Mx[8], Mx[8]);
}

typedef struct {
    float M0[3], M1[3]; /* rows of the 2x3 matrix J*W */
    float tx, ty, tz;   /* clamped view-space point used in J */
    float xmul, ymul;   /* 0 where the guard-band clamp was active */
    float a, b, c;      /* raw cov2D (no dilation) */
} cov2d_aux;

/* EWA projection of Sigma; Appendix A.1 step 4 */
static inline void cov2d_project(const float* pview, const float* cov6, const float* view,
                                 float focal_x, float focal_y, float tanfovx, float tanfovy,
                                 cov2d_aux* o) {
    float tz = pview[2];
    float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
    float txtz = pview[0] / tz, tytz = pview[1] / tz;
    o->xmul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    o->ymul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    float tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    float ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
    o->tx = tx; o->ty = ty; o->tz = tz;
    float tz2 = tz * tz;
    float J00 = focal_x / tz;
    float J02 = -(focal_x * tx) / tz2;
    float J11 = focal_y / tz;
    float J12 = -(focal_y * ty) / tz2;
    /* W[i][j] = view[4*j+i] */
    for (int j = 0; j < 3; j++) {
        float W0j = view[4 * j + 0], W1j = view[4 * j + 1], W2j = view[4 * j + 2];
        o->M0[j] = fmaf(J02, W2j, J00 * W0j);
        o->M1[j] = fmaf(J12, W2j, J11 * W1j);
    }
    const float* M0 = o->M0; const float* M1 = o->M1;
    float S00 = cov6[0], S01 = cov6[1], S02 = cov6[2], S11 = cov6[3], S12 = cov6[4], S22 = cov6[5];
    float v0 = dot3_fma(S00, M0[0], S01, M0[1], S02, M0[2]);
    float v1 = dot3_fma(S01, M0[0], S11, M0[1], S12, M0[2]);
    float v2 = dot3_fma(S02, M0[0], S12, M0[1], S22, M0[2]);
    float w0 = dot3_fma(S00, M1[0], S01, M1[1], S02, M1[2]);
    float w1 = dot3_fma(S01, M1[0], S11, M1[1], S12, M1[2]);
    float w2 = dot3_fma(S02, M1[0], S12, M1[1], S22, M1[2]);
    o->a = dot3_fma(M0[0], v0, M0[1], v1, M0[2], v2);
    o->b = dot3_fma(M1[0], v0, M1[1], v1, M1[2], v2);
    o->c = dot3_fma(M1[0], w0, M1[1], w1, M1[2], w2);
}

/* Canonical evaluation of  -0.5*(cx*dx*dx + cz*dy*dy) - cy*dx*dy  (Appendix A.2): the FMA-contracted
 * form of the upstream expression; edge-on flat Gaussians make the three terms cancel, so the op order
 * is part of the contract (the CUDA kernels replay it bit-for-bit; only exp() may differ by ulps). */
static inline float quad_power(const float* co, float dx, float dy) {
    float m1 = co[0] * dx;
    float m2 = m1 * dx;
    float m3 = co[2] * dy;
    float t = fmaf(m3, dy, m2);
    float h = -0.5f * t;
    float m4 = co[1] * dx;
    return fmaf(-m4, dy, h);
}

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* float -> int32 with the device's cvt.rzi.s32.f32 semantics: truncate toward zero, saturate to [INT32_MIN, INT32_MAX],
 * NaN -> 0.  A C cast is undefined outside the int32 range (x86 returns INT32_MIN at either end), so a radius beyond
 * int32 or a rect bound of a centre far off-screen would otherwise disagree with the kernels for no reason of theirs. */
int32_t gmso_f2i_sat(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return INT32_MAX;
    if (v <= -2147483648.0f) return INT32_MIN;
    return (int32_t)v;
}

static inline void get_rect(float px, float py, int radius, int gx, int gy, int* rmin, int* rmax) {
    float r = (float)radius;
    rmin[0] = imin(gx, imax(0, gmso_f2i_sat((px - r) / (float)GMSO_BLOCK)));
    rmin[1] = imin(gy, imax(0, gmso_f2i_sat((py - r) / (float)GMSO_BLOCK)));
    rmax[0] = imin(gx, imax(0, gmso_f2i_sat((px + r + (float)(GMSO_BLOCK - 1)) / (float)GMSO_BLOCK)));
    rmax[1] = imin(gy, imax(0, gmso_f2i_sat((py + r + (float)(GMSO_BLOCK - 1)) / (float)GMSO_BLOCK)));
}

/* SH basis, utils/sh_utils.py:74-100 (degree <= 3) */
static inline void sh_basis(int deg, float x, float y, float z, float* B) {
    B[0] = SH_C0;
    if (deg > 0) {
        B[1] = -SH_C1 * y; B[2] = SH_C1 * z; B[3] = -SH_C1 * x;
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            B[4] = SH_C2[0] * xy; B[5] = SH_C2[1] * yz;
            B[6] = SH_C2[2] * (2.0f * zz - xx - yy);
            B[7] = SH_C2[3] * xz; B[8] = SH_C2[4] * (xx - yy);
            if (deg > 2) {
                B[9] = SH_C3[0] * y * (3.0f * xx - yy);
                B[10] = SH_C3[1] * xy * z;
                B[11] = SH_C3[2] * y * (4.0f * zz - xx - yy);
                B[12] = SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
                B[13] = SH_C3[4] * x * (4.0f * zz - xx - yy);
                B[14] = SH_C3[5] * z * (xx - yy);
                B[15] = SH_C3[6] * x * (xx - 3.0f * yy);
            }
        }
    }
}

/* d(basis)/d(dir) */
static inline void sh_basis_grad(int deg, float x, float y, float z, float* Bx, float* By, float* Bz) {
    for (int k = 0; k < 16; k++) { Bx[k] = 0.f; By[k] = 0.f; Bz[k] = 0.f; }
    if (deg > 0) {
        By[1] = -SH_C1; Bz[2] = SH_C1; Bx[3] = -SH_C1;
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            Bx[4] = SH_C2[0] * y; By[4] = SH_C2[0] * x;
            By[5] = SH_C2[1] * z; Bz[5] = SH_C2[1] * y;
            Bx[6] = SH_C2[2] * (-2.f * x); By[6] = SH_C2[2] * (-2.f * y); Bz[6] = SH_C2[2] * (4.f * z);
            Bx[7] = SH_C2[3] * z; Bz[7] = SH_C2[3] * x;
            Bx[8] = SH_C2[4] * (2.f * x); By[8] = SH_C2[4] * (-2.f * y);
            if (deg > 2) {
                Bx[9] = SH_C3[0] * 6.f * xy; By[9] = SH_C3[0] * (3.f * xx - 3.f * yy);
                Bx[10] = SH_C3[1] * yz; By[10] = SH_C3[1] * xz; Bz[10] = SH_C3[1] * xy;
                Bx[11] = SH_C3[2] * (-2.f * xy); By[11] = SH_C3[2] * (4.f * zz - xx - 3.f * yy);
                Bz[11] = SH_C3[2] * 8.f * yz;
                Bx[12] = SH_C3[3] * (-6.f * xz); By[12] = SH_C3[3] * (-6.f * yz);
                Bz[12] = SH_C3[3] * (6.f * zz - 3.f * xx - 3.f * yy);
                Bx[13] = SH_C3[4] * (4.f * zz - 3.f * xx - yy); By[13] = SH_C3[4] * (-2.f * xy);
                Bz[13] = SH_C3[4] * 8.f * xz;
                Bx[14] = SH_C3[5] * 2.f * xz; By[14] = SH_C3[5] * (-2.f * yz); Bz[14] = SH_C3[5] * (xx - yy);
                Bx[15] = SH_C3[6] * (3.f * xx - 3.f * yy); By[15] = SH_C3[6] * (-6.f * xy);
            }
        }
    }
}

/* =====================================================================
 * A.1  preprocess forward.  Any output pointer may be NULL except radii.
 * ===================================================================== */
int gmso_preprocess_forward(const gmso_settings* s,
                            const float* means3D,      /* [P,3] */
                            const float* scales,       /* [P,3] or NULL */
                            const float* rotations,    /* [P,4] or NULL */
                            const float* cov3D_precomp,/* [P,6] or NULL */
                            const float* opacities,    /* [P] */
                            const float* shs,          /* [P,M,3] or NULL */
                            const float* colors_precomp,/* [P,3] or NULL */
                            int32_t* radii, float* means2D /*[P,2]*/, float* depths,
                            float* cov3Ds /*[P,6]*/, float* conic_opacity /*[P,4]*/,
                            float* rgb /*[P,3]*/, uint8_t* clamped /*[P,3]*/,
                            uint32_t* tiles_touched, int32_t* rects /*[P,4] xmin,ymin,xmax,ymax*/) {
    const int P = s->P, W = s->W, H = s->H;
    const int gx = (W + GMSO_BLOCK - 1) / GMSO_BLOCK, gy = (H + GMSO_BLOCK - 1) / GMSO_BLOCK;
    const float focal_x = (float)W / (2.0f * s->tanfovx);
    const float focal_y = (float)H / (2.0f * s->tanfovy);
    if (s->D < 0 || s->D > 3) return -1;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        radii[i] = 0;
        if (tiles_touched) tiles_touched[i] = 0;
        if (rects) { rects[4 * i] = rects[4 * i + 1] = rects[4 * i + 2] = rects[4 * i + 3] = 0; }
        if (means2D) { means2D[2 * i] = 0.f; means2D[2 * i + 1] = 0.f; }
        if (depths) depths[i] = 0.f;
        if (conic_opacity) { for (int k = 0; k < 4; k++) conic_opacity[4 * i + k] = 0.f; }
        if (rgb) { for (int k = 0; k < 3; k++) rgb[3 * i + k] = 0.f; }
        if (clamped) { for (int k = 0; k < 3; k++) clamped[3 * i + k] = 0; }
        if (cov3Ds) { for (int k = 0; k < 6; k++) cov3Ds[6 * i + k] = 0.f; }

        const float x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        float pview[3];
        xform4x3(s->viewmatrix, x, y, z, pview);
        if (pview[2] <= 0.2f) continue; /* near cull (in_frustum) */
        float phom[4];
        xform4x4(s->projmatrix, x, y, z, phom);
        float pw = 1.0f / (phom[3] + 0.0000001f);
        float pprojx = phom[0] * pw, pprojy = phom[1] * pw;

        float cov6[6];
        if (cov3D_precomp) {
            for (int k = 0; k < 6; k++) cov6[k] = cov3D_precomp[6 * i + k];
        } else {
            cov3d_from_scale_rot(scales + 3 * i, s->scale_modifier, rotations + 4 * i, cov6);
        }
        if (cov3Ds) { for (int k = 0; k < 6; k++) cov3Ds[6 * i + k] = cov6[k]; }

        cov2d_aux ca;
        cov2d_project(pview, cov6, s->viewmatrix, focal_x, focal_y, s->tanfovx, s->tanfovy, &ca);
        float a = ca.a, b = ca.b, c = ca.c;
        const float h_var = 0.3f;
        float det_cov = fmaf(a, c, -(b * b));
        a = a + h_var; c = c + h_var;
        float det = fmaf(a, c, -(b * b));
        if (det == 0.0f) continue;
        float h_scale = 1.0f;
        if (s->antialiasing) h_scale = sqrtf(fmaxf(0.000025f, det_cov / det));
        float det_inv = 1.f / det;
        float conx = c * det_inv, cony = -b * det_inv, conz = a * det_inv;

        float mid = 0.5f * (a + c);
        float disc = sqrtf(fmaxf(0.1f, fmaf(mid, mid, -det)));
        float lambda1 = mid + disc, lambda2 = mid - disc;
        int my_radius = gmso_f2i_sat(ceilf(3.f * sqrtf(fmaxf(lambda1, lambda2))));
        float pixx = fmaf(pprojx + 1.0f, (float)W, -1.0f) * 0.5f;
        float pixy = fmaf(pprojy + 1.0f, (float)H, -1.0f) * 0.5f;
        int rmin[2], rmax[2];
        get_rect(pixx, pixy, my_radius, gx, gy, rmin, rmax);
        int area = (rmax[0] - rmin[0]) * (rmax[1] - rmin[1]);
        if (area == 0) continue;

        if (rgb) {
            if (colors_precomp) {
                for (int k = 0; k < 3; k++) rgb[3 * i + k] = colors_precomp[3 * i + k];
            } else {
                float dx = x - s->campos[0], dy = y - s->campos[1], dz = z - s->campos[2];
                float len = sqrtf(dx * dx + dy * dy + dz * dz);
                dx /= len; dy /= len; dz /= len;
                float B[16];
                sh_basis(s->D, dx, dy, dz, B);
                int nc = (s->D + 1) * (s->D + 1);
                const float* sh = shs + (size_t)i * s->M * 3;
                for (int ch = 0; ch < 3; ch++) {
                    float acc = 0.f;
                    for (int k = 0; k < nc; k++) acc += B[k] * sh[3 * k + ch];
                    acc += 0.5f;
                    if (clamped) clamped[3 * i + ch] = (acc < 0.f) ? 1 : 0;
                    rgb[3 * i + ch] = fmaxf(acc, 0.f);
                }
            }
        }
        if (depths) depths[i] = pview[2];
        radii[i] = my_radius;
        if (means2D) { means2D[2 * i] = pixx; means2D[2 * i + 1] = pixy; }
        if (conic_opacity) {
            conic_opacity[4 * i] = conx; conic_opacity[4 * i + 1] = cony; conic_opacity[4 * i + 2] = conz;
            conic_opacity[4 * i + 3] = opacities[i] * h_scale;
        }
        if (tiles_touched) tiles_touched[i] = (uint32_t)area;
        if (rects) { rects[4 * i] = rmin[0]; rects[4 * i + 1] = rmin[1]; rects[4 * i + 2] = rmax[0]; rects[4 * i + 3] = rmax[1]; }
    }
    return 0;
}

/* number of key bits for the tile id (upstream getHigherMsb) */
int gmso_tile_bits(int ntiles) {
    uint32_t n = (uint32_t)ntiles;
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step; else msb -= step;
    }
    if (n >> msb) msb++;
    return (int)msb;
}

/* =====================================================================
 * Binning: inclusive scan, duplicate-with-keys, stable sort, tile ranges.
 * offsets[P] is written; returns N.  If keys_sorted/point_list are NULL only
 * the count is produced.  Capacity of the key arrays must be >= N.
 * ===================================================================== */
int64_t gmso_bin(const gmso_settings* s, const int32_t* radii, const float* depths,
                 const int32_t* rects, const uint32_t* tiles_touched, uint32_t* offsets,
                 uint64_t* keys_sorted, uint32_t* point_list, int32_t* ranges /*[T,2]*/,
                 int64_t capacity) {
    const int P = s->P;
    const int gx = (s->W + GMSO_BLOCK - 1) / GMSO_BLOCK, gy = (s->H + GMSO_BLOCK - 1) / GMSO_BLOCK;
    uint64_t run = 0;
    for (int i = 0; i < P; i++) { run += tiles_touched[i]; offsets[i] = (uint32_t)run; }
    int64_t N = (int64_t)run;
    if (!keys_sorted || !point_list) return N;
    if (N > capacity) return -N;
    uint64_t* k0 = keys_sorted; uint32_t* v0 = point_list;
    uint64_t* k1 = (uint64_t*)malloc(sizeof(uint64_t) * (size_t)(N > 0 ? N : 1));
    uint32_t* v1 = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(N > 0 ? N : 1));
    /* duplicateWithKeys */
#pragma omp parallel for schedule(dynamic, 1024)
    for (int i = 0; i < P; i++) {
        if (radii[i] <= 0) continue;
        uint32_t off = (i == 0) ? 0u : offsets[i - 1];
        uint32_t dbits; memcpy(&dbits, &depths[i], 4);
        for (int y = rects[4 * i + 1]; y < rects[4 * i + 3]; y++)
            for (int x = rects[4 * i]; x < rects[4 * i + 2]; x++) {
                uint64_t key = (uint64_t)(uint32_t)(y * gx + x);
                key = (key << 32) | dbits;
                k0[off] = key; v0[off] = (uint32_t)i; off++;
            }
    }
    /* stable LSD radix sort, 16 bits per pass, over bits [0, 32+tile_bits) */
    int nbits = 32 + gmso_tile_bits(gx * gy);
    int npass = (nbits + 15) / 16;
    uint32_t* hist = (uint32_t*)malloc(sizeof(uint32_t) * 65536);
    uint64_t* ka = k0; uint32_t* va = v0; uint64_t* kb = k1; uint32_t* vb = v1;
    for (int p = 0; p < npass; p++) {
        int shift = 16 * p;
        memset(hist, 0, sizeof(uint32_t) * 65536);
        for (int64_t j = 0; j < N; j++) hist[(ka[j] >> shift) & 0xFFFF]++;
        uint32_t sum = 0;
        for (int d = 0; d < 65536; d++) { uint32_t c = hist[d]; hist[d] = sum; sum += c; }
        for (int64_t j = 0; j < N; j++) {
            uint32_t d = (uint32_t)((ka[j] >> shift) & 0xFFFF);
            uint32_t pos = hist[d]++;
            kb[pos] = ka[j]; vb[pos] = va[j];
        }
        uint64_t* tk = ka; ka = kb; kb = tk;
        uint32_t* tv = va; va = vb; vb = tv;
    }
    if (ka != k0) { memcpy(k0, ka, sizeof(uint64_t) * (size_t)N); memcpy(v0, va, sizeof(uint32_t) * (size_t)N); }
    free(hist); free(k1); free(v1);
    /* identifyTileRanges */
    if (ranges) {
        memset(ranges, 0, sizeof(int32_t) * 2 * (size_t)(gx * gy));
        for (int64_t j = 0; j < N; j++) {
            uint32_t t = (uint32_t)(k0[j] >> 32);
            if (j == 0) ranges[2 * t] = 0;
            else {
                uint32_t tp = (uint32_t)(k0[j - 1] >> 32);
                if (tp != t) { ranges[2 * tp + 1] = (int32_t)j; ranges[2 * t] = (int32_t)j; }
            }
            if (j == N - 1) ranges[2 * t + 1] = (int32_t)N;
        }
    }
    return N;
}

/* =====================================================================
 * A.2 composite forward (one pixel at a time, the tile's list front to back).
 * ambiguous[px] (optional) is set when a skip/stop decision was within a few
 * ulp of its threshold, i.e. a different-but-valid exp() could flip it.
 * ===================================================================== */
int gmso_composite_forward(const gmso_settings* s, const int32_t* ranges, const uint32_t* point_list,
                           const float* means2D, const float* rgb, const float* conic_opacity,
                           const float* depths,
                           float* out_color /*[3,H,W]*/, float* final_T /*[H,W]*/,
                           int32_t* n_contrib /*[H,W]*/, float* out_invdepth /*[H,W] or NULL*/,
                           uint8_t* ambiguous /*[H,W] or NULL*/) {
    const int W = s->W, H = s->H;
    const int gx = (W + GMSO_BLOCK - 1) / GMSO_BLOCK, gy = (H + GMSO_BLOCK - 1) / GMSO_BLOCK;
    long long st0 = 0, st1 = 0, st2 = 0, st3 = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : st0, st1, st2, st3)
    for (int tile = 0; tile < gx * gy; tile++) {
        if (tile % g_tile_stride) continue;
        int tx0 = (tile % gx) * GMSO_BLOCK, ty0 = (tile / gx) * GMSO_BLOCK;
        int r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        uint8_t* qhit = (uint8_t*)calloc((size_t)(r1 - r0) + 1, 1);
        for (int py = ty0; py < ty0 + GMSO_BLOCK && py < H; py++)
            for (int px = tx0; px < tx0 + GMSO_BLOCK && px < W; px++) {
                const int quad = ((py - ty0) >> 3) * 2 + ((px - tx0) >> 3);
                float T = 1.0f, C[3] = {0.f, 0.f, 0.f}, Dacc = 0.f;
                int contributor = 0, last = 0; uint8_t amb = 0;
                float pfx = (float)px, pfy = (float)py;
                for (int j = r0; j < r1; j++) {
                    contributor++; st0++;
                    uint32_t g = point_list[j];
                    float dx = means2D[2 * g] - pfx, dy = means2D[2 * g + 1] - pfy;
                    const float* co = conic_opacity + 4 * g;
                    float power = quad_power(co, dx, dy);
                    if (power > 0.0f) continue;
                    float alpha = fminf(0.99f, co[3] * expf(power));
                    if (fabsf(alpha - 1.0f / 255.0f) < 4e-6f * (1.0f / 255.0f) + 1e-9f) amb = 1;
                    if (alpha < 1.0f / 255.0f) continue;
                    float test_T = T * (1.f - alpha);
                    if (fabsf(test_T - 0.0001f) < 1e-9f) amb = 1;
                    if (test_T < 0.0001f) break;
                    float w = alpha * T;
                    for (int ch = 0; ch < 3; ch++) C[ch] += rgb[3 * g + ch] * w;
                    Dacc += (1.f / depths[g]) * w;
                    T = test_T;
                    last = contributor;
                    st1++; qhit[j - r0] |= (uint8_t)(1u << quad);
                }
                size_t pix = (size_t)py * W + px;
                final_T[pix] = T; n_contrib[pix] = last;
                for (int ch = 0; ch < 3; ch++) out_color[(size_t)ch * H * W + pix] = C[ch] + T * s->bg[ch];
                if (out_invdepth) out_invdepth[pix] = Dacc;
                if (ambiguous) ambiguous[pix] = amb;
            }
        for (int j = 0; j < r1 - r0; j++) {
            if (qhit[j]) st3++;
            st2 += ((qhit[j] >> 0) & 1) + ((qhit[j] >> 1) & 1) + ((qhit[j] >> 2) & 1) + ((qhit[j] >> 3) & 1);
        }
        free(qhit);
    }
    g_stats[0] = st0; g_stats[1] = st1; g_stats[2] = st2; g_stats[3] = st3;
    return 0;
}

/* =====================================================================
 * A.3 composite backward.  Accumulates in double (this is the checker).
 * Outputs are per-Gaussian: dL_dmean2D[P,2] (NDC-scaled: *0.5W / *0.5H),
 * dL_dconic[P,3] = (xx, xy-HALF-convention, yy), dL_dopacity[P] (w.r.t.
 * conic_opacity.w), dL_dcolor[P,3], dL_dinvdepth[P].
 * ===================================================================== */
int gmso_composite_backward(const gmso_settings* s, const int32_t* ranges, const uint32_t* point_list,
                            const float* means2D, const float* rgb, const float* conic_opacity,
                            const float* depths, const float* final_T, const int32_t* n_contrib,
                            const float* dL_dpix /*[3,H,W]*/, const float* dL_dinvdepth_pix /*[H,W] or NULL*/,
                            double* dL_dmean2D, double* dL_dconic, double* dL_dopacity,
                            double* dL_dcolor, double* dL_dinvdepth) {
    const int W = s->W, H = s->H, P = s->P;
    const int gx = (W + GMSO_BLOCK - 1) / GMSO_BLOCK, gy = (H + GMSO_BLOCK - 1) / GMSO_BLOCK;
    memset(dL_dmean2D, 0, sizeof(double) * 2 * (size_t)P);
    memset(dL_dconic, 0, sizeof(double) * 3 * (size_t)P);
    memset(dL_dopacity, 0, sizeof(double) * (size_t)P);
    memset(dL_dcolor, 0, sizeof(double) * 3 * (size_t)P);
    memset(dL_dinvdepth, 0, sizeof(double) * (size_t)P);
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
    /* serial over tiles: per-Gaussian accumulators are shared between tiles */
    int nth = gmso_num_threads();
    (void)nth;
#pragma omp parallel
    {
        double* l_m = (double*)calloc((size_t)P * 10, sizeof(double));
#pragma omp for schedule(dynamic, 1)
        for (int tile = 0; tile < gx * gy; tile++) {
            if (tile % g_tile_stride) continue;
            int tx0 = (tile % gx) * GMSO_BLOCK, ty0 = (tile / gx) * GMSO_BLOCK;
            int r0 = ranges[2 * tile];
            for (int py = ty0; py < ty0 + GMSO_BLOCK && py < H; py++)
                for (int px = tx0; px < tx0 + GMSO_BLOCK && px < W; px++) {
                    size_t pix = (size_t)py * W + px;
                    float Tfin = final_T[pix];
                    float T = Tfin;
                    int last = n_contrib[pix];
                    float dpix[3];
                    for (int ch = 0; ch < 3; ch++) dpix[ch] = dL_dpix[(size_t)ch * H * W + pix];
                    float dinv = dL_dinvdepth_pix ? dL_dinvdepth_pix[pix] : 0.f;
                    float accum_rec[3] = {0.f, 0.f, 0.f}, last_color[3] = {0.f, 0.f, 0.f};
                    float accum_inv = 0.f, last_inv = 0.f, last_alpha = 0.f;
                    float bg_dot = s->bg[0] * dpix[0] + s->bg[1] * dpix[1] + s->bg[2] * dpix[2];
                    float pfx = (float)px, pfy = (float)py;
                    for (int j = r0 + last - 1; j >= r0; j--) {
                        uint32_t g = point_list[j];
                        float dx = means2D[2 * g] - pfx, dy = means2D[2 * g + 1] - pfy;
                        const float* co = conic_opacity + 4 * g;
                        float power = quad_power(co, dx, dy);
                        if (power > 0.0f) continue;
                        float G = expf(power);
                        float alpha = fminf(0.99f, co[3] * G);
                        if (alpha < 1.0f / 255.0f) continue;
                        T = T / (1.f - alpha);
                        float dch = alpha * T;
                        float dL_dalpha = 0.f;
                        double* acc = l_m + (size_t)g * 10;
                        for (int ch = 0; ch < 3; ch++) {
                            float c = rgb[3 * g + ch];
                            accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                            last_color[ch] = c;
                            dL_dalpha += (c - accum_rec[ch]) * dpix[ch];
                            acc[6 + ch] += (double)(dch * dpix[ch]);
                        }
                        {
                            float invd = 1.f / depths[g];
                            accum_inv = last_alpha * last_inv + (1.f - last_alpha) * accum_inv;
                            last_inv = invd;
                            dL_dalpha += (invd - accum_inv) * dinv;
                            acc[9] += (double)(dch * dinv);
                        }
                        dL_dalpha *= T;
                        last_alpha = alpha;
                        dL_dalpha += (-Tfin / (1.f - alpha)) * bg_dot;
                        float dL_dG = co[3] * dL_dalpha;
                        float gdx = G * dx, gdy = G * dy;
                        float dG_ddelx = -gdx * co[0] - gdy * co[1];
                        float dG_ddely = -gdy * co[2] - gdx * co[1];
                        acc[0] += (double)(dL_dG * dG_ddelx * ddelx_dx);
                        acc[1] += (double)(dL_dG * dG_ddely * ddely_dy);
                        acc[2] += (double)(-0.5f * gdx * dx * dL_dG);
                        acc[3] += (double)(-0.5f * gdx * dy * dL_dG);
                        acc[4] += (double)(-0.5f * gdy * dy * dL_dG);
                        acc[5] += (double)(G * dL_dalpha);
                    }
                }
        }
#pragma omp critical
        {
            for (int g = 0; g < P; g++) {
                const double* a = l_m + (size_t)g * 10;
                dL_dmean2D[2 * g] += a[0]; dL_dmean2D[2 * g + 1] += a[1];
                dL_dconic[3 * g] += a[2]; dL_dconic[3 * g + 1] += a[3]; dL_dconic[3 * g + 2] += a[4];
                dL_dopacity[g] += a[5];
                dL_dcolor[3 * g] += a[6]; dL_dcolor[3 * g + 1] += a[7]; dL_dcolor[3 * g + 2] += a[8];
                dL_dinvdepth[g] += a[9];
            }
        }
        free(l_m);
    }
    return 0;
}

/* =====================================================================
 * A.3 in float64, with a per-element error budget.
 *
 * ref64[P,10]: the per-Gaussian sums of gmso_composite_backward (same order: mean2D x/y NDC-scaled, conic xx/xy(half)/yy,
 * opacity, rgb, inverse depth), every per-pair quantity evaluated in double.  The blend decisions (which splats blend at a
 * pixel, n_contrib) are the fp32 forward's, and G = exp() in double of the canonical fp32 power (quad_power) -- the
 * operation is defined by the fp32 forward, whose decisions the kernels reproduce bit for bit outside threshold-ambiguous
 * pixels; a float64 power would weigh other pixels for edge-on slivers.  dx, dy are the fp32 differences both sides form.
 * alpha = min(0.99f, op * G); T is the double front-to-back product over the blended splats (not recovered by division from
 * the fp32 final_T), the background term uses the double final T, and dL/dalpha, the colour-behind recurrence and the
 * moment terms are double.  Like the two functions above, it covers only the tiles gmso_set_tile_stride selects.
 *
 * budget[P,10]: a first-order bound, derived from the operation sequence of the fp32 kernels (gms_bwd_pair, gms_red_flush,
 * gms_bwd_commit), on |any correct fp32 implementation - ref64|.  u = 2^-24.  Every term is bounded through its absolute
 * value, per blended (pixel, splat) pair:
 *     cd   = |c . dL/dC| summed per channel (+ |invd * dL/dD|),   bgd = sum_ch |bg_ch * dL/dC_ch|,
 *     Babs = the colour-behind recurrence on absolute values:  Babs <- alpha * cd + (1 - alpha) * Babs,
 *     |q|  = G * (T * (cd + Babs) + T_final * bgd / (1 - alpha)),
 *     mean2D x: op * W/2 * |q| * (|conx dx| + |cony dy|),   mean2D y: op * H/2 * |q| * (|conz dy| + |cony dx|),
 *     conic:    op/2 * |q| * (dx^2, |dx dy|, dy^2),          opacity: |q|,    rgb / inverse depth: alpha * T * |dL/dC|, |dL/dD|.
 * With m = that magnitude, the pair's share is u * (C0 + K_p) * m and each Gaussian adds u * (CSUM + n_quads_i) * sum m:
 *   C0 = 24, the longest chain of one pair's own roundings:  G = ex2.approx(power * log2e):  <= 2^-22 (4 u) for ex2, and
 *        |power| * (1 + 0.23) u <= 6.8 u for the argument (blending needs G >= 1/255, |power| <= ln 255; 0.23 u is the
 *        rounding of log2e), alpha = op * G: 1 -> alpha within 12 u;  c . dL/dC: 4 (three / four FMAs);  c - Bdot, * T, the
 *        FMA with the background term: 3;  * G: 1 (+ G's 12);  the moment products before the sum (q dy, + of the lane's two
 *        pixels, dx * (dx * sq)): 3;  w = alpha * T and the dL/dC products: alpha's 12 + 2.  12 + 1 + 4 + 3 + 3 + 1 = 24.
 *   K_p  = sum over the pixel's blended splats l of (CSTEP + CALPHA * a_l):  the transmittance in front of splat j is
 *        recovered as final_T * prod_{l >= j} rcp(1 - alpha_l), with final_T the fp32 forward product: per splat 2 u in the
 *        forward (1 - alpha, *) and 4 u in the recovery (1 - alpha, rcp.approx <= 1 ulp = 2 u, *); the alpha of a splat in
 *        FRONT of j enters T_j with its own error (12 u) times alpha / (1 - alpha) (behind j it cancels between the forward
 *        product and the recovery).  Bdot for a splat behind j costs 2 u (FMA, *) plus alpha's 12 u times
 *        max(1, alpha / (1 - alpha)).  T_j's and Bdot_j's splat sets are disjoint (in front / behind), so
 *        CSTEP = 6 + 14 = 20 and CALPHA = 12, with a_l = alpha_l / (1 - alpha_l) (0 where alpha is clamped to 0.99f:
 *        the same constant on both sides).  Unlike a plain count k this keeps the 1 / (1 - alpha) amplification of nearly
 *        opaque splats.
 *   CSUM = 22, the summation:  each quad adds its 64 pixels as two pixels per lane (1) and a serial 32-term row sum in two
 *        16-chains joined at the end (15 + 1) in its shared-memory panel, then the commit's products (<= 5: conx * s, the
 *        FMA with cony * s, * op, * W/2).  n_quads_i = the number of 8x8 quads in which Gaussian i blends at any pixel: the
 *        float atomics add one partial sum per (quad, splat) pair in any order, a chain of at most n_quads_i.
 * Threshold-ambiguous pixels (ambiguous[px], see gmso_composite_forward) get an ALLOWANCE: an fp32 implementation with
 * another exp() may take the other decision for a splat f whose alpha lies in the band around 1/255 (blended or not), or
 * not stop at the splat f that ended the pixel.  Each such f is a flip candidate; for each one, to first order:
 *   - f itself gains or loses its whole term: its full magnitude m_f;
 *   - a blended splat j behind f sees T_j, and every blended j sees T_final, scaled by (1 - alpha_f) or its inverse, a
 *     relative change <= r_f = alpha_f / (1 - alpha_f) (alpha_f for a candidate that does not blend in the forward):
 *     r_f * m_j for j behind f (its T-terms, colour terms included), r_f * G_j T_final bgd / (1 - alpha_j) for j in front;
 *   - a blended splat j in front of f sees its colour behind change by the product of (1 - alpha) between them times
 *     alpha_f (c_f - B_f) . dL/dC, so T_j Bdot_j moves by <= alpha_f (cd_f + cmax) T_f / (1 - alpha_j), T_f the
 *     transmittance in front of f and cmax the largest cd at the pixel (|B| <= cmax for any set of decisions),
 * each carried through the moment factors of the magnitude above.  These are added to the budgets (nothing is exempted).
 * A candidate that does not blend in the forward is a pair the other implementation adds, with its own roundings: its
 * magnitude also enters the rounding shares above, at C0 + K_p + CSTEP + CALPHA * a_f (the pixel's chain one splat
 * longer), and the summation share through n_quads_i, which counts the quads of candidates too.
 * amb_share[i] = the largest share of any component's budget of Gaussian i that comes from such allowances.
 * A Gaussian that blends at no pixel and decides at no ambiguous pixel has ref64 = budget = 0: exactly zero is required.
 * ===================================================================== */
#define GMSO_U (1.0 / 16777216.0)
#define GMSO_C0 24.0
#define GMSO_CSTEP 20.0
#define GMSO_CALPHA 12.0
#define GMSO_CSUM 22.0
#define GMSO_NACC 41    /* per Gaussian and thread: ref 10, (C0+K)*m 10, m 10, allowance 10, n_quads 1 */

typedef struct {
    uint32_t g;
    int blend;          /* blends in the fp32 forward; 0: a decision candidate at an ambiguous pixel */
    int flip;           /* a decision another exp() may take the other way (ambiguous pixels only) */
    double dx, dy, G, alpha, T, cd, Babs;
} gmso_e64;

/* the ten term magnitudes of a pair whose |dL/dalpha * G| is qa and whose colour weight alpha * T is w */
static inline void gmso_mag64(const float* co, const gmso_e64* x, double qa, double w, const double* dpx, double dinv,
                              double hW, double hH, double* m) {
    const double cx = co[0], cy = co[1], cz = co[2], op = co[3], dx = x->dx, dy = x->dy;
    m[0] = op * hW * qa * (fabs(cx * dx) + fabs(cy * dy));
    m[1] = op * hH * qa * (fabs(cz * dy) + fabs(cy * dx));
    m[2] = 0.5 * op * qa * dx * dx;
    m[3] = 0.5 * op * qa * fabs(dx * dy);
    m[4] = 0.5 * op * qa * dy * dy;
    m[5] = qa;
    for (int ch = 0; ch < 3; ch++) m[6 + ch] = w * fabs(dpx[ch]);
    m[9] = w * fabs(dinv);
}

int gmso_composite_backward64(const gmso_settings* s, const int32_t* ranges, const uint32_t* point_list,
                              const float* means2D, const float* rgb, const float* conic_opacity,
                              const float* depths, const int32_t* n_contrib, const uint8_t* ambiguous,
                              const float* dL_dpix /*[3,H,W]*/, const float* dL_dinvdepth_pix /*[H,W] or NULL*/,
                              double* ref64 /*[P,10]*/, double* budget /*[P,10]*/, double* amb_share /*[P]*/) {
    const int W = s->W, H = s->H, P = s->P;
    const int gx = (W + GMSO_BLOCK - 1) / GMSO_BLOCK, gy = (H + GMSO_BLOCK - 1) / GMSO_BLOCK;
    const double hW = (double)(0.5f * W), hH = (double)(0.5f * H);
    const double amax = (double)0.99f;
    const double bgc[3] = {s->bg[0], s->bg[1], s->bg[2]};
    int maxlen = 1;
    for (int t = 0; t < gx * gy; t++) maxlen = imax(maxlen, ranges[2 * t + 1] - ranges[2 * t]);
    double* tot = (double*)calloc((size_t)P * GMSO_NACC, sizeof(double));
    if (!tot) return -1;
#pragma omp parallel
    {
        double* l = (double*)calloc((size_t)P * GMSO_NACC, sizeof(double));
        gmso_e64* e = (gmso_e64*)malloc(sizeof(gmso_e64) * (size_t)maxlen);
        uint8_t* qhit = (uint8_t*)malloc((size_t)maxlen);
#pragma omp for schedule(dynamic, 1)
        for (int tile = 0; tile < gx * gy; tile++) {
            if (tile % g_tile_stride) continue;
            const int tx0 = (tile % gx) * GMSO_BLOCK, ty0 = (tile / gx) * GMSO_BLOCK;
            const int r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            memset(qhit, 0, (size_t)maxlen);
            for (int py = ty0; py < ty0 + GMSO_BLOCK && py < H; py++)
                for (int px = tx0; px < tx0 + GMSO_BLOCK && px < W; px++) {
                    const size_t pix = (size_t)py * W + px;
                    const int quad = ((py - ty0) >> 3) * 2 + ((px - tx0) >> 3);
                    const int last = n_contrib[pix], amb = ambiguous[pix] != 0;
                    const float pfx = (float)px, pfy = (float)py;
                    /* the fp32 forward's decisions; at an ambiguous pixel also the band candidates and the stopping splat */
                    int n = 0;
                    const int lim = amb ? r1 - r0 : last;
                    float T32 = 1.0f;
                    for (int jj = 0; jj < lim; jj++) {
                        const uint32_t g = point_list[r0 + jj];
                        const float dx = means2D[2 * g] - pfx, dy = means2D[2 * g + 1] - pfy;
                        const float* co = conic_opacity + 4 * g;
                        const float power = quad_power(co, dx, dy);
                        if (power > 0.0f) continue;
                        const float a32 = fminf(0.99f, co[3] * expf(power));
                        /* the forward's ambiguity tests, decision by decision */
                        const int aband = amb && fabsf(a32 - 1.0f / 255.0f) < 4e-6f * (1.0f / 255.0f) + 1e-9f;
                        const int blend = a32 >= 1.0f / 255.0f && jj < last;
                        const int stop = a32 >= 1.0f / 255.0f && jj >= last;     /* the splat the forward stopped at */
                        const float test_T = T32 * (1.f - a32);
                        const int tband = amb && a32 >= 1.0f / 255.0f && fabsf(test_T - 0.0001f) < 1e-9f;
                        if (blend) T32 = test_T;
                        if (!blend && !((aband || tband) && (stop || a32 < 1.0f / 255.0f))) {
                            if (stop) break;
                            continue;
                        }
                        gmso_e64* x = e + n++;
                        x->g = g; x->blend = blend;
                        x->flip = aband | (tband && blend ? 2 : 0) | (tband && stop ? 4 : 0);
                        x->dx = dx; x->dy = dy;
                        x->G = exp((double)power);
                        x->alpha = fmin(amax, (double)co[3] * x->G);
                        qhit[jj] |= (uint8_t)(1u << quad);
                        if (stop) break;
                    }
                    if (n == 0) continue;
                    double T = 1.0, K = 0.0;
                    for (int k = 0; k < n; k++) {
                        e[k].T = T;
                        if (!e[k].blend) continue;
                        const double a = e[k].alpha;
                        K += GMSO_CSTEP + (a < amax ? GMSO_CALPHA * a / (1.0 - a) : 0.0);
                        T *= 1.0 - a;
                    }
                    const double Tfin = T;
                    double dpx[3], bgdot = 0.0, bgabs = 0.0;
                    for (int ch = 0; ch < 3; ch++) {
                        dpx[ch] = dL_dpix[(size_t)ch * H * W + pix];
                        bgdot += bgc[ch] * dpx[ch];
                        bgabs += fabs(bgc[ch] * dpx[ch]);
                    }
                    const double dinv = dL_dinvdepth_pix ? dL_dinvdepth_pix[pix] : 0.0;
                    double B = 0.0, Babs = 0.0, cmax = 0.0;
                    for (int k = n - 1; k >= 0; k--) {
                        const uint32_t g = e[k].g;
                        const float* co = conic_opacity + 4 * g;
                        const double cx = co[0], cy = co[1], cz = co[2], op = co[3];
                        const double dx = e[k].dx, dy = e[k].dy, G = e[k].G, a = e[k].alpha, Tk = e[k].T;
                        const double invd = 1.0 / (double)depths[g];
                        double cdp = invd * dinv, cd = fabs(invd * dinv);
                        for (int ch = 0; ch < 3; ch++) {
                            cdp += (double)rgb[3 * g + ch] * dpx[ch];
                            cd += fabs((double)rgb[3 * g + ch] * dpx[ch]);
                        }
                        e[k].cd = cd; e[k].Babs = Babs;
                        cmax = fmax(cmax, cd);
                        if (!e[k].blend) continue;
                        const double dLa = Tk * (cdp - B) - Tfin * bgdot / (1.0 - a);
                        const double q = dLa * G;
                        const double t[10] = {op * hW * q * (-cx * dx - cy * dy), op * hH * q * (-cz * dy - cy * dx),
                                              -0.5 * op * q * dx * dx, -0.5 * op * q * dx * dy, -0.5 * op * q * dy * dy, q,
                                              a * Tk * dpx[0], a * Tk * dpx[1], a * Tk * dpx[2], a * Tk * dinv};
                        double m[10];
                        gmso_mag64(co, e + k, G * (Tk * (cd + Babs) + Tfin * bgabs / (1.0 - a)), a * Tk, dpx, dinv, hW, hH, m);
                        double* acc = l + (size_t)g * GMSO_NACC;
                        for (int c = 0; c < 10; c++) {
                            acc[c] += t[c];
                            acc[10 + c] += (GMSO_C0 + K) * m[c];
                            acc[20 + c] += m[c];
                        }
                        B = a * cdp + (1.0 - a) * B;
                        Babs = a * cd + (1.0 - a) * Babs;
                    }
                    /* allowances for the flip candidates of an ambiguous pixel */
                    for (int f = 0; f < n; f++) {
                        if (!e[f].flip) continue;
                        const double af = e[f].alpha, Tf = e[f].T;
                        const double rf = e[f].blend ? af / (1.0 - af) : af;
                        for (int k = 0; k < n; k++) {
                            const gmso_e64* x = e + k;
                            if (k != f && !x->blend) continue;
                            const double a = x->alpha, G = x->G, Tk = x->T;
                            const double full = G * (Tk * (x->cd + x->Babs) + Tfin * bgabs / (1.0 - a));
                            double qa = 0.0, w = 0.0;
                            if (e[f].flip & 5) {          /* f alone blends or not */
                                if (k == f) { qa = full; w = a * Tk; }
                                else if (k > f) { qa = rf * full; w = rf * a * Tk; }
                                else qa = G * (af * (e[f].cd + cmax) * Tf + rf * Tfin * bgabs) / (1.0 - a);
                            }
                            if (e[f].flip & 2) {          /* the pixel stops at f: f and everything behind it drop out */
                                if (k >= f) { qa += full; w += a * Tk; }
                                else qa += G * Tf * (cmax + bgabs) / (1.0 - a);
                            }
                            double m[10];
                            gmso_mag64(conic_opacity + 4 * x->g, x, qa, w, dpx, dinv, hW, hH, m);
                            double* acc = l + (size_t)x->g * GMSO_NACC;
                            for (int c = 0; c < 10; c++) acc[30 + c] += m[c];
                            if (k == f && !x->blend) {
                                /* the pair another implementation adds carries its own roundings and enters the sums */
                                double mo[10];
                                gmso_mag64(conic_opacity + 4 * x->g, x, full, a * Tk, dpx, dinv, hW, hH, mo);
                                const double Kf = K + GMSO_CSTEP + (a < amax ? GMSO_CALPHA * a / (1.0 - a) : 0.0);
                                for (int c = 0; c < 10; c++) {
                                    acc[10 + c] += (GMSO_C0 + Kf) * mo[c];
                                    acc[20 + c] += mo[c];
                                }
                            }
                        }
                    }
                }
            for (int jj = 0; jj < r1 - r0; jj++) {
                const uint8_t h = qhit[jj];
                if (h) l[(size_t)point_list[r0 + jj] * GMSO_NACC + 40] += (h & 1) + ((h >> 1) & 1) + ((h >> 2) & 1) + ((h >> 3) & 1);
            }
        }
#pragma omp critical
        {
            for (size_t k = 0; k < (size_t)P * GMSO_NACC; k++) tot[k] += l[k];
        }
        free(l); free(e); free(qhit);
    }
    for (int i = 0; i < P; i++) {
        const double* a = tot + (size_t)i * GMSO_NACC;
        double share = 0.0;
        for (int c = 0; c < 10; c++) {
            const double b = GMSO_U * (a[10 + c] + (GMSO_CSUM + a[40]) * a[20 + c]) + a[30 + c];
            ref64[10 * i + c] = a[c];
            budget[10 * i + c] = b;
            if (b > 0.0) share = fmax(share, a[30 + c] / b);
        }
        amb_share[i] = share;
    }
    free(tot);
    return 0;
}

/* =====================================================================
 * A.2 in float64, with a per-pixel error budget.
 *
 * ref[5,H,W]: colour r, g, b, inverse depth and final T of every pixel, on the blend decisions of the fp32 forward above
 * (gmso_composite_forward: which splats blend, where the pixel stops), every value in double: G = exp() in double of the
 * canonical fp32 power (quad_power: bit-identical in the kernels, so power <= 0 is never in doubt and edge-on slivers stay
 * defined), alpha = min(0.99f, op * G), the T product, w = alpha * T, the colour and inverse-depth sums and the T_final * bg
 * term.  The inputs are the fp32 per-splat record: means2D, conic / opacity, rgb and the fp32 1 / depth the record holds.
 *
 * budget[5,H,W]: a first-order bound on |any correct fp32 implementation - ref|, from the operation sequence of the kernels
 * (k_composite_fwd2: scalar FMAs; k_composite_fwd3: the same roundings on float2 pairs) and of the fp32 oracle (no
 * contraction, expf).  u = 2^-24.  Per blended splat l, in list order:
 *   G    = ex2.approx.ftz(power * log2e): 4 u (2^-22) for ex2, |power| * 1.23 u for the rounded argument and log2e, as in
 *          gmso_composite_backward64 (the oracle's expf is within 1 ulp);
 *   alpha = op * G: + u, so da_l = alpha_l * ea_l with ea_l = 4 u + 1.23 u |power| + u; the clamp min(0.99f, .) is 1-Lipschitz
 *          and needs no allowance, and da_l = 0 where op * G * (1 - ea_l) >= 0.99f (both sides take the constant);
 *   1 - alpha: da_l / (1 - alpha_l) relative (alpha's error amplified by alpha / (1 - alpha)) + u for the subtraction;
 *   T_{l+1} = T_l * (1 - alpha_l): eT_{l+1} = eT_l + da_l / (1 - alpha_l) + 2 u (relative, eT_1 = 0);
 *   w_l = alpha_l * T_l: da_l / alpha_l + eT_l + u;
 *   colour: C_l = fma(c_l, w_l, C_{l-1}) (the oracle: a product and a sum, one more u): |c_l| w_l (da_l / alpha_l + eT_l + 2 u)
 *          + min(u * sum_{k <= l} |c_k| w_k, |c_l| w_l), the rounding of the partial sum: at most half an ulp of it, and at most
 *          the term itself, since the old sum is a representable candidate of the rounding (a faint splat that a long sum
 *          absorbs costs no more than its own term); inverse depth alike;
 *   final:  fma(T_final, bg, C) (the oracle: two roundings): |bg| T_final (eT_final + 2 u) + min(u (sum_l |c_l| w_l +
 *          |bg| T_final), |bg| T_final);
 *   final T: T_final * eT_final.
 * rgb_tol > 0 adds rgb_tol * (|c_l| + 1) * w_l per blended splat: the colour record is then known to that relative and
 * absolute tolerance only (a caller without the kernels' own record).
 *
 * Decision candidates, from the same bounds (nothing is a fixed band):
 *   skip:  |alpha - 1/255| <= da: another exp() may blend a splat the fp32 forward skips, or skip one it blends;
 *   stop:  |T (1 - alpha) - 1e-4| <= T (1 - alpha) (eT + da / (1 - alpha) + 2 u + Wf), Wf = the sum over the skip candidates
 *          in front of r' = alpha / (1 - alpha) (blended) or alpha (skipped): a flipped skip in front scales this T by
 *          (1 - alpha)^(-+1).  Tested at every splat the forward reaches with alpha >= 1/255 and, hypothetically, at the
 *          skip candidates it passes.
 * Each candidate f adds an ALLOWANCE, to first order what flipping it changes (T_f, the transmittance in front of f; S_f, the
 * sum of |c_l| w_l over the blended splats behind f):
 *   (A) f alone blends or not: alpha_f T_f |c_f| + r'_f (S_f + T_final |bg|); final T: r'_f T_final;
 *   (B) the pixel stops at f (it went on in the forward): sum_{l >= f} |c_l| w_l + |bg| (T_f - T_final); final T: T_f - T_final;
 *   (C) the pixel goes on past the splat it stopped at: at most all the remaining contributions, T_f (cmax + |bg|) with cmax
 *       the largest |c| of the tile's list; final T: T_f.
 * adm[H,W,8]: the admissible n_contrib values: the fp32 forward's, then those the candidates produce ((A): f's position or the
 * blended one before it; (B): the blended one before f; (C): f's position and every later one the pixel may still blend, by
 * walking the list with the upper bound of T).  -1 pads; -2 in the last slot: more than fit, any value >= adm[0] is admitted.
 * cand[H,W] = 1 where the pixel has a candidate.
 * qhit[N]: bit q of a list position set when its splat blends at some in-image pixel of 8x8 quad q of its tile (the fp32
 * decisions); qcand[N]: bit q set when a candidate of a pixel of quad q may change whether that splat blends there.
 * Like the functions above, it covers only the tiles gmso_set_tile_stride selects.
 * ===================================================================== */
#define GMSO_NADM 8

typedef struct {
    int pos, before, blend, stop, skipc, stopc;      /* before: the position of the blended splat in front (0: none) */
    double a, da, T, eT, W, w, c[3], invd;
} gmso_f64;

static inline void gmso_adm_add(int32_t* adm, int v) {
    for (int k = 0; k < GMSO_NADM; k++) {
        if (adm[k] == v || adm[k] == -2) return;
        if (adm[k] == -1) { adm[k] = v; return; }
    }
    adm[GMSO_NADM - 1] = -2;
}

int gmso_composite_forward64(const gmso_settings* s, const int32_t* ranges, const uint32_t* point_list,
                             const float* means2D, const float* rgb, const float* conic_opacity, const float* depths,
                             double rgb_tol, double* ref /*[5,H,W]*/, double* budget /*[5,H,W]*/, double* allowance /*[5,H,W]*/,
                             int32_t* adm /*[H,W,8]*/, uint8_t* cand /*[H,W]*/, uint8_t* qhit /*[N]*/, uint8_t* qcand /*[N]*/) {
    const int W = s->W, H = s->H;
    const size_t HW = (size_t)W * H;
    const int gx = (W + GMSO_BLOCK - 1) / GMSO_BLOCK, gy = (H + GMSO_BLOCK - 1) / GMSO_BLOCK;
    const double u = GMSO_U, amax = (double)0.99f, thr = (double)(1.0f / 255.0f), tstop = (double)0.0001f;
    const double bgc[3] = {s->bg[0], s->bg[1], s->bg[2]};
    const double bga[3] = {fabs(bgc[0]), fabs(bgc[1]), fabs(bgc[2])};
    int maxlen = 1;
    for (int t = 0; t < gx * gy; t++) maxlen = imax(maxlen, ranges[2 * t + 1] - ranges[2 * t]);
    memset(ref, 0, sizeof(double) * 5 * HW);
    memset(budget, 0, sizeof(double) * 5 * HW);
    memset(allowance, 0, sizeof(double) * 5 * HW);
    memset(cand, 0, HW);
    for (size_t k = 0; k < GMSO_NADM * HW; k++) adm[k] = -1;
#pragma omp parallel
    {
        gmso_f64* e = (gmso_f64*)malloc(sizeof(gmso_f64) * (size_t)maxlen);
#pragma omp for schedule(dynamic, 1)
        for (int tile = 0; tile < gx * gy; tile++) {
            if (tile % g_tile_stride) continue;
            const int tx0 = (tile % gx) * GMSO_BLOCK, ty0 = (tile / gx) * GMSO_BLOCK;
            const int r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            double cmax[3] = {0.0, 0.0, 0.0}, dmax = 0.0;
            for (int j = r0; j < r1; j++) {
                const uint32_t g = point_list[j];
                for (int ch = 0; ch < 3; ch++) cmax[ch] = fmax(cmax[ch], fabs((double)rgb[3 * g + ch]));
                dmax = fmax(dmax, fabs((double)(1.f / depths[g])));
            }
            for (int j = r0; j < r1; j++) { qhit[j] = 0; qcand[j] = 0; }
            for (int py = ty0; py < ty0 + GMSO_BLOCK && py < H; py++)
                for (int px = tx0; px < tx0 + GMSO_BLOCK && px < W; px++) {
                    const size_t pix = (size_t)py * W + px;
                    const uint8_t qb = (uint8_t)(1u << (((py - ty0) >> 3) * 2 + ((px - tx0) >> 3)));
                    const float pfx = (float)px, pfy = (float)py;
                    int32_t* ad = adm + GMSO_NADM * pix;
                    /* front to back: the fp32 forward's decisions (T32), the double values, the rounding bounds */
                    float T32 = 1.0f;
                    double T = 1.0, eT = 0.0, Wf = 0.0, C[3] = {0.0, 0.0, 0.0}, D = 0.0, Cabs[3] = {0.0, 0.0, 0.0}, Dabs = 0.0;
                    double errC[3] = {0.0, 0.0, 0.0}, errD = 0.0;
                    int n = 0, last = 0, stop_at = -1;
                    for (int jj = 0; jj < r1 - r0; jj++) {
                        const uint32_t g = point_list[r0 + jj];
                        const float dx = means2D[2 * g] - pfx, dy = means2D[2 * g + 1] - pfy;
                        const float* co = conic_opacity + 4 * g;
                        const float power = quad_power(co, dx, dy);
                        if (power > 0.0f) continue;
                        const float a32 = fminf(0.99f, co[3] * expf(power));
                        const double G = exp((double)power), opG = (double)co[3] * G, a = fmin(amax, opG);
                        const double ea = 4.0 * u + 1.23 * u * fabs((double)power) + u;
                        const double da = opG * (1.0 - ea) >= amax ? 0.0 : a * ea;
                        const int skipc = fabs(a - thr) <= da;
                        const int blendable = a32 >= 1.0f / 255.0f;
                        if (!blendable && !skipc) continue;
                        const float test32 = T32 * (1.f - a32);
                        const int stop = blendable && test32 < 0.0001f;
                        const int blend = blendable && !stop;
                        gmso_f64* x = e + n++;
                        x->pos = jj + 1; x->before = last; x->blend = blend; x->stop = stop; x->skipc = skipc;
                        x->a = a; x->da = da; x->T = T; x->eT = eT; x->W = Wf; x->w = 0.0;
                        for (int ch = 0; ch < 3; ch++) x->c[ch] = rgb[3 * g + ch];
                        x->invd = (double)(1.f / depths[g]);
                        const double tT = T * (1.0 - a);
                        x->stopc = fabs(tT - tstop) <= tT * (eT + da / (1.0 - a) + 2.0 * u + Wf);
                        if (skipc) Wf += blend ? a / (1.0 - a) : a;
                        if (blend) {
                            const double w = a * T, ew = da / a + eT + 2.0 * u;
                            x->w = w;
                            for (int ch = 0; ch < 3; ch++) {
                                const double cw = fabs(x->c[ch]) * w;
                                C[ch] += x->c[ch] * w;
                                Cabs[ch] += cw;
                                errC[ch] += cw * ew + fmin(u * Cabs[ch], cw) + rgb_tol * (fabs(x->c[ch]) + 1.0) * w;
                            }
                            D += x->invd * w;
                            Dabs += fabs(x->invd) * w;
                            errD += fabs(x->invd) * w * ew + fmin(u * Dabs, fabs(x->invd) * w);
                            T = tT;
                            eT += da / (1.0 - a) + 2.0 * u;
                            T32 = test32;
                            last = jj + 1;
                            qhit[r0 + jj] |= qb;
                        }
                        if (stop) { stop_at = n - 1; break; }
                    }
                    const double Tfin = T;
                    ad[0] = last;
                    for (int ch = 0; ch < 3; ch++) {
                        ref[ch * HW + pix] = C[ch] + Tfin * bgc[ch];
                        budget[ch * HW + pix] = errC[ch] + bga[ch] * Tfin * (eT + 2.0 * u) + fmin(u * (Cabs[ch] + bga[ch] * Tfin), bga[ch] * Tfin);
                    }
                    ref[3 * HW + pix] = D;
                    budget[3 * HW + pix] = errD;
                    ref[4 * HW + pix] = Tfin;
                    budget[4 * HW + pix] = Tfin * eT;
                    /* allowances: S[k] = sum over the blended splats from entry k on of |c| w (and invd w) */
                    double S[3] = {0.0, 0.0, 0.0}, Sd = 0.0, al[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
                    int any = 0;
                    for (int k = n - 1; k >= 0; k--) {
                        gmso_f64* f = e + k;
                        const double Sb[3] = {S[0], S[1], S[2]}, Sdb = Sd;     /* behind f */
                        for (int ch = 0; ch < 3; ch++) S[ch] += fabs(f->c[ch]) * f->w;
                        Sd += fabs(f->invd) * f->w;
                        const int before = f->before;
                        if (f->skipc && !f->stop) {                             /* (A) */
                            const double r = f->blend ? f->a / (1.0 - f->a) : f->a;
                            for (int ch = 0; ch < 3; ch++) al[ch] += f->a * f->T * fabs(f->c[ch]) + r * (Sb[ch] + Tfin * bga[ch]);
                            al[3] += f->a * f->T * fabs(f->invd) + r * Sdb;
                            al[4] += r * Tfin;
                            if (f->blend && f->pos == last) gmso_adm_add(ad, before);
                            if (!f->blend && f->pos > last) gmso_adm_add(ad, f->pos);
                            qcand[r0 + f->pos - 1] |= qb;
                            any = 1;
                        }
                        if (f->stopc && (f->blend || (!f->stop && f->skipc))) {   /* (B) */
                            for (int ch = 0; ch < 3; ch++) al[ch] += S[ch] + bga[ch] * (f->T - Tfin);
                            al[3] += Sd;
                            al[4] += f->T - Tfin;
                            gmso_adm_add(ad, before);
                            for (int m = k; m < n; m++) if (e[m].blend) qcand[r0 + e[m].pos - 1] |= qb;
                            any = 1;
                        }
                        if (k == stop_at && (f->stopc || f->skipc)) {         /* (C) */
                            for (int ch = 0; ch < 3; ch++) al[ch] += f->T * (cmax[ch] + bga[ch]);
                            al[3] += f->T * dmax;
                            al[4] += f->T;
                            any = 1;
                            /* the positions the pixel may still blend: walk on with the upper bound of T */
                            const double rel = 1.0 + f->eT + f->W + 2.0 * u;
                            double Thi = f->skipc ? f->T * rel : 0.0;
                            if (f->stopc) {
                                gmso_adm_add(ad, f->pos);
                                qcand[r0 + f->pos - 1] |= qb;
                                Thi = fmax(Thi, f->T * (1.0 - f->a + f->da) * rel);
                            }
                            for (int jj = f->pos; jj < r1 - r0; jj++) {
                                const uint32_t g = point_list[r0 + jj];
                                const float dx = means2D[2 * g] - pfx, dy = means2D[2 * g + 1] - pfy;
                                const float* co = conic_opacity + 4 * g;
                                const float power = quad_power(co, dx, dy);
                                if (power > 0.0f) continue;
                                const double G = exp((double)power), opG = (double)co[3] * G, a = fmin(amax, opG);
                                const double ea = 4.0 * u + 1.23 * u * fabs((double)power) + u;
                                const double da = opG * (1.0 - ea) >= amax ? 0.0 : a * ea;
                                if (a + da < thr) continue;
                                const int canskip = a - da < thr;
                                const int canblend = Thi * (1.0 - a + da) >= tstop;
                                if (canblend) { gmso_adm_add(ad, jj + 1); qcand[r0 + jj] |= qb; }
                                if (!canskip && !canblend) break;
                                if (!canskip) Thi *= 1.0 - a + da;
                            }
                        }
                    }
                    for (int c = 0; c < 5; c++) { allowance[c * HW + pix] = al[c]; budget[c * HW + pix] += al[c]; }
                    cand[pix] = (uint8_t)any;
                }
        }
        free(e);
    }
    return 0;
}

/* =====================================================================
 * A.4 preprocess backward (computeCov2D backward + projection + SH + cov3D).
 * Inputs are the per-Gaussian gradients from the composite backward (float).
 * ===================================================================== */
int gmso_preprocess_backward(const gmso_settings* s, const int32_t* radii,
                             const float* means3D, const float* scales, const float* rotations,
                             const float* cov3D_precomp, const float* opacities, const float* shs,
                             const float* colors_precomp, const float* cov3Ds, const uint8_t* clamped,
                             const float* dL_dmean2D /*[P,2]*/, const float* dL_dconic /*[P,3]*/,
                             const float* dL_dopacity_in /*[P] wrt conic_opacity.w*/,
                             const float* dL_dcolor /*[P,3]*/, const float* dL_dinvdepth /*[P] or NULL*/,
                             float* dL_dmeans3D /*[P,3]*/, float* dL_dcov3D /*[P,6]*/,
                             float* dL_dsh /*[P,M,3] or NULL*/, float* dL_dcolors_precomp /*[P,3] or NULL*/,
                             float* dL_dscale /*[P,3] or NULL*/, float* dL_drot /*[P,4] or NULL*/,
                             float* dL_dopacity_out /*[P]*/) {
    const int P = s->P, W = s->W, H = s->H;
    const float focal_x = (float)W / (2.0f * s->tanfovx);
    const float focal_y = (float)H / (2.0f * s->tanfovy);
    const float* view = s->viewmatrix; const float* proj = s->projmatrix;
    (void)colors_precomp; (void)cov3D_precomp;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        for (int k = 0; k < 3; k++) dL_dmeans3D[3 * i + k] = 0.f;
        for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = 0.f;
        if (dL_dsh) memset(dL_dsh + (size_t)i * s->M * 3, 0, sizeof(float) * 3 * (size_t)s->M);
        if (dL_dcolors_precomp) for (int k = 0; k < 3; k++) dL_dcolors_precomp[3 * i + k] = 0.f;
        if (dL_dscale) for (int k = 0; k < 3; k++) dL_dscale[3 * i + k] = 0.f;
        if (dL_drot) for (int k = 0; k < 4; k++) dL_drot[4 * i + k] = 0.f;
        dL_dopacity_out[i] = 0.f;
        if (radii[i] <= 0) continue;

        const float x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        const float* cov6 = cov3Ds + 6 * i;
        float pview[3];
        xform4x3(view, x, y, z, pview);
        cov2d_aux ca;
        cov2d_project(pview, cov6, view, focal_x, focal_y, s->tanfovx, s->tanfovy, &ca);
        const float h_var = 0.3f;
        float a0 = ca.a, b = ca.b, c0 = ca.c;       /* raw */
        float a = a0 + h_var, c = c0 + h_var;        /* dilated */
        float det_cov = a0 * c0 - b * b;
        float det = a * c - b * b;

        float dcx = dL_dconic[3 * i], dcy = dL_dconic[3 * i + 1], dcz = dL_dconic[3 * i + 2];
        float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;

        /* opacity (and antialiasing compensation) */
        float dop = dL_dopacity_in[i];
        if (s->antialiasing) {
            float ratio = det_cov / det;
            float h_scale = sqrtf(fmaxf(0.000025f, ratio));
            dL_dopacity_out[i] = dop * h_scale;
            if (ratio > 0.000025f) {
                /* d L / d ratio, ratio = det_cov/det; both depend on raw a0,b,c0 */
                float dL_dratio = dop * opacities[i] / (2.f * h_scale);
                float inv_det = 1.f / det;
                /* d ratio / d a0 = (c0*det - det_cov*c)/det^2 etc. */
                dL_da += dL_dratio * (c0 * det - det_cov * c) * inv_det * inv_det;
                dL_dc += dL_dratio * (a0 * det - det_cov * a) * inv_det * inv_det;
                dL_db += dL_dratio * (-2.f * b * det + 2.f * b * det_cov) * inv_det * inv_det;
            }
        } else {
            dL_dopacity_out[i] = dop;
        }

        float denom = det;
        float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        if (denom2inv != 0.f) {
            dL_da += denom2inv * (-c * c * dcx + 2.f * b * c * dcy + (denom - a * c) * dcz);
            dL_dc += denom2inv * (-a * a * dcz + 2.f * a * b * dcy + (denom - a * c) * dcx);
            dL_db += denom2inv * 2.f * (b * c * dcx - (denom + 2.f * b * b) * dcy + a * b * dcz);
        }
        const float* M0 = ca.M0; const float* M1 = ca.M1;
        float g6[6];
        g6[0] = M0[0] * M0[0] * dL_da + M0[0] * M1[0] * dL_db + M1[0] * M1[0] * dL_dc;
        g6[3] = M0[1] * M0[1] * dL_da + M0[1] * M1[1] * dL_db + M1[1] * M1[1] * dL_dc;
        g6[5] = M0[2] * M0[2] * dL_da + M0[2] * M1[2] * dL_db + M1[2] * M1[2] * dL_dc;
        g6[1] = 2.f * M0[0] * M0[1] * dL_da + (M0[0] * M1[1] + M0[1] * M1[0]) * dL_db + 2.f * M1[0] * M1[1] * dL_dc;
        g6[2] = 2.f * M0[0] * M0[2] * dL_da + (M0[0] * M1[2] + M0[2] * M1[0]) * dL_db + 2.f * M1[0] * M1[2] * dL_dc;
        g6[4] = 2.f * M0[2] * M0[1] * dL_da + (M0[1] * M1[2] + M0[2] * M1[1]) * dL_db + 2.f * M1[1] * M1[2] * dL_dc;
        for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = g6[k];

        /* dL/dM = [2 da M0 + db M1 ; 2 dc M1 + db M0] * Sigma */
        float S[9] = {cov6[0], cov6[1], cov6[2], cov6[1], cov6[3], cov6[4], cov6[2], cov6[4], cov6[5]};
        float u0[3], u1[3], dM0[3], dM1[3];
        for (int j = 0; j < 3; j++) {
            u0[j] = 2.f * dL_da * M0[j] + dL_db * M1[j];
            u1[j] = 2.f * dL_dc * M1[j] + dL_db * M0[j];
        }
        for (int j = 0; j < 3; j++) {
            dM0[j] = u0[0] * S[0 * 3 + j] + u0[1] * S[1 * 3 + j] + u0[2] * S[2 * 3 + j];
            dM1[j] = u1[0] * S[0 * 3 + j] + u1[1] * S[1 * 3 + j] + u1[2] * S[2 * 3 + j];
        }
        float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
        for (int j = 0; j < 3; j++) {
            float W0j = view[4 * j + 0], W1j = view[4 * j + 1], W2j = view[4 * j + 2];
            dJ00 += dM0[j] * W0j; dJ02 += dM0[j] * W2j;
            dJ11 += dM1[j] * W1j; dJ12 += dM1[j] * W2j;
        }
        float tz = 1.f / ca.tz, tz2 = tz * tz, tz3 = tz2 * tz;
        float dL_dtx = ca.xmul * -focal_x * tz2 * dJ02;
        float dL_dty = ca.ymul * -focal_y * tz2 * dJ12;
        float dL_dtz = -focal_x * tz2 * dJ00 - focal_y * tz2 * dJ11 +
                       (2.f * focal_x * ca.tx) * tz3 * dJ02 + (2.f * focal_y * ca.ty) * tz3 * dJ12;
        if (dL_dinvdepth) dL_dtz -= dL_dinvdepth[i] / (pview[2] * pview[2]);
        /* transformVec4x3Transpose: dmean = W^T dt */
        float dmx = view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
        float dmy = view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
        float dmz = view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;

        /* mean2D -> mean3D through the projection */
        float phom[4];
        xform4x4(proj, x, y, z, phom);
        float m_w = 1.0f / (phom[3] + 0.0000001f);
        float mul1 = phom[0] * m_w * m_w;
        float mul2 = phom[1] * m_w * m_w;
        float g2x = dL_dmean2D[2 * i], g2y = dL_dmean2D[2 * i + 1];
        dmx += (proj[0] * m_w - proj[3] * mul1) * g2x + (proj[1] * m_w - proj[3] * mul2) * g2y;
        dmy += (proj[4] * m_w - proj[7] * mul1) * g2x + (proj[5] * m_w - proj[7] * mul2) * g2y;
        dmz += (proj[8] * m_w - proj[11] * mul1) * g2x + (proj[9] * m_w - proj[11] * mul2) * g2y;

        /* colour */
        if (shs && dL_dsh) {
            float dx = x - s->campos[0], dy = y - s->campos[1], dz = z - s->campos[2];
            float len = sqrtf(dx * dx + dy * dy + dz * dz);
            float ux = dx / len, uy = dy / len, uz = dz / len;
            float B[16], Bx[16], By[16], Bz[16];
            sh_basis(s->D, ux, uy, uz, B);
            sh_basis_grad(s->D, ux, uy, uz, Bx, By, Bz);
            int nc = (s->D + 1) * (s->D + 1);
            const float* sh = shs + (size_t)i * s->M * 3;
            float* dsh = dL_dsh + (size_t)i * s->M * 3;
            float ddx = 0.f, ddy = 0.f, ddz = 0.f;
            for (int ch = 0; ch < 3; ch++) {
                float g = dL_dcolor[3 * i + ch] * (clamped[3 * i + ch] ? 0.f : 1.f);
                for (int k = 0; k < nc; k++) {
                    dsh[3 * k + ch] = B[k] * g;
                    ddx += Bx[k] * sh[3 * k + ch] * g;
                    ddy += By[k] * sh[3 * k + ch] * g;
                    ddz += Bz[k] * sh[3 * k + ch] * g;
                }
            }
            /* through v/|v| */
            float dotp = ux * ddx + uy * ddy + uz * ddz;
            dmx += (ddx - ux * dotp) / len;
            dmy += (ddy - uy * dotp) / len;
            dmz += (ddz - uz * dotp) / len;
        } else if (dL_dcolors_precomp) {
            for (int k = 0; k < 3; k++) dL_dcolors_precomp[3 * i + k] = dL_dcolor[3 * i + k];
        }
        dL_dmeans3D[3 * i] = dmx; dL_dmeans3D[3 * i + 1] = dmy; dL_dmeans3D[3 * i + 2] = dmz;

        /* cov3D -> scale, rotation */
        if (scales && rotations && dL_dscale && dL_drot) {
            float R[9];
            const float* q = rotations + 4 * i;
            quat_to_R(q, R);
            float mod = s->scale_modifier;
            float sv[3] = {mod * scales[3 * i], mod * scales[3 * i + 1], mod * scales[3 * i + 2]};
            float Mx[9];
            for (int r = 0; r < 3; r++) for (int cc = 0; cc < 3; cc++) Mx[3 * r + cc] = R[3 * r + cc] * sv[cc];
            float dS[9] = {g6[0], 0.5f * g6[1], 0.5f * g6[2], 0.5f * g6[1], g6[3], 0.5f * g6[4],
                           0.5f * g6[2], 0.5f * g6[4], g6[5]};
            float dMx[9];
            for (int r = 0; r < 3; r++) for (int cc = 0; cc < 3; cc++)
                dMx[3 * r + cc] = 2.f * (dS[3 * r] * Mx[cc] + dS[3 * r + 1] * Mx[3 + cc] + dS[3 * r + 2] * Mx[6 + cc]);
            float dR[9];
            for (int cc = 0; cc < 3; cc++) {
                float acc = 0.f;
                for (int r = 0; r < 3; r++) { acc += R[3 * r + cc] * dMx[3 * r + cc]; dR[3 * r + cc] = dMx[3 * r + cc] * sv[cc]; }
                dL_dscale[3 * i + cc] = acc * mod;
            }
            float qr = q[0], qx = q[1], qy = q[2], qz = q[3];
            dL_drot[4 * i + 0] = 2.f * (-qz * dR[1] + qy * dR[2] + qz * dR[3] - qx * dR[5] - qy * dR[6] + qx * dR[7]);
            dL_drot[4 * i + 1] = 2.f * (-2.f * qx * (dR[4] + dR[8]) + qy * (dR[1] + dR[3]) + qz * (dR[2] + dR[6]) + qr * (dR[7] - dR[5]));
            dL_drot[4 * i + 2] = 2.f * (-2.f * qy * (dR[0] + dR[8]) + qx * (dR[1] + dR[3]) + qr * (dR[2] - dR[6]) + qz * (dR[5] + dR[7]));
            dL_drot[4 * i + 3] = 2.f * (-2.f * qz * (dR[0] + dR[4]) + qr * (dR[3] - dR[1]) + qx * (dR[2] + dR[6]) + qy * (dR[5] + dR[7]));
        }
    }
    return 0;
}

/* markVisible / checkFrustum (R10) */
int gmso_mark_visible(const gmso_settings* s, const float* means3D, uint8_t* present) {
    for (int i = 0; i < s->P; i++) {
        float pview[3];
        xform4x3(s->viewmatrix, means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2], pview);
        present[i] = pview[2] > 0.2f ? 1 : 0;
    }
    return 0;
}
