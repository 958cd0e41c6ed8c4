// gms_composite_bwd.cuh -- per-tile compositing, backward (see gms_composite_common.cuh for the decomposition).
//
// Both kernels walk a quad's splats back to front, one (quad, splat) pair at a time through gms_bwd_pair (scalar fp32 for the
// lane's two pixels, which share their column and therefore dx), accumulate per-lane the 9 (10 with a depth loss) moment sums
//     sum q dx, sum q dy, sum q dx^2, sum q dx dy, sum q dy^2, sum q, sum w dL/dC[3] (, sum w dL/dD),   q = dL/dalpha * G,
// reduce them over the warp through a shared-memory panel (three splats per row-sum pass, no shuffles), and issue three
// vector reductions (red.global.add.v4.f32 x2 + .v2) per blended (quad, splat) pair -- instead of the stock 9-10 scalar
// atomics per blended (pixel, splat) pair.
// Restructuring that removes per-pixel state and branches:
//  * the stock recurrence keeps (last_alpha, last_color, accum_rec); here the "colour behind" B is advanced at the END
//    of a splat's step,  B <- alpha*c + (1-alpha)*B , one step earlier.  B only ever enters as (c - B) . dL/dC with dL/dC
//    fixed per pixel, so the lane carries the scalar Bdot = B . dL/dC instead:  Bdot <- alpha*(c . dL/dC) + (1-alpha)*Bdot;
//  * a pixel that does not blend a splat (beyond n_contrib, power > 0, alpha < 1/255) uses alpha_eff = 0: then
//    T/(1-0) = T, Bdot <- 0*x + 1*Bdot = Bdot exactly, and its moment contributions are masked to 0 -- no divergent branch.
//
// k_composite_bwd5  default: walks the SURVIVOR LIST the forward pass wrote for this quad (k_composite_fwd2<true>): every
//                   staged splat is one that blended, so there is no culling test, no vote, and 32 useful pairs per round.
// k_composite_bwd3  predecessor (A/B, and the fallback when a forward ran without lists): streams the whole tile list and
//                   re-derives the survivors with the ellipse-vs-rectangle test.
#pragma once
#include "gms_composite_common.cuh"

struct GmsSlabB {              // one copy of each staged splat (gms_slabb_store)
    float4 a[GMS_WB];          // x, y, conx, -cony
    float4 b[GMS_WB];          // conz, opacity, r, g
    float2 c[GMS_WB];          // b, 1/depth
    int id[GMS_WB];
    int pos[GMS_WB];
    float part[GMS_WB][12];    // the splat's warp-reduced moment sums (gms_red_flush)
};

__device__ __forceinline__ void gms_slabb_store(GmsSlabB& S, int lane, const float4& ra, const float4& rb, const float4& rc) {
    S.a[lane] = make_float4(ra.x, ra.y, ra.z, -ra.w);
    S.b[lane] = rb;
    S.c[lane] = make_float2(rc.x, rc.y);
}

// Deferred warp reduction: every lane parks its NV partial sums of up to three splats in a [3*NV][32] shared-memory panel
// (row stride 36 floats: conflict-free column stores and conflict-free 128-bit row loads); lane r then adds up row r
// (8 LDS.128 + 31 FADD for three splats at once) and writes S.part.  The slab indices of the pending splats are shifted into
// pj one byte at a time, so the newest is in the low byte; lane r's splat is byte (pending - 1 - r / NV), at bit `sh`.
constexpr int GMS_RED_STRIDE = 36;

__device__ __forceinline__ void gms_red_flush(const float* red, float (*part)[12], int pj, int nrows, int lane, int sh, int ri) {
    __syncwarp();
    if (lane < nrows) {
        const float4* row = reinterpret_cast<const float4*>(red + lane * GMS_RED_STRIDE);
        const float4 a = row[0];
        float s0 = a.x + a.y, s1 = a.z + a.w;
#pragma unroll
        for (int c = 1; c < 8; c++) { const float4 t = row[c]; s0 += t.x; s1 += t.z; s0 += t.y; s1 += t.w; }
        part[(pj >> sh) & 31][ri] = s0 + s1;
    }
    __syncwarp();
}

// Panel bookkeeping of one warp: the column the next splat's sums go to, and the pending splats.
template <int NV>
struct GmsPanel {
    float* col;                // panel + pend * NV * GMS_RED_STRIDE + lane, panel = this warp's [3*NV][GMS_RED_STRIDE] floats
    int pend, pj;              // pending splats, their slab indices (a byte each)
    int sh3, ri;               // lane r sums row r = value ri of pending splat r / NV: byte 2 - r / NV when three are pending

    __device__ __forceinline__ GmsPanel(float* panel, int lane) : col(panel + lane), pend(0), pj(0) {
        sh3 = 8 * (2 - lane / NV); ri = lane % NV;
        asm volatile("" : "+r"(sh3), "+r"(ri));
    }
    // the splat in slab slot j has written its column: advance, and reduce once three splats are pending
    __device__ __forceinline__ void push(int j, float (*part)[12], int lane) {
        pj = pj * 256 + j;
        col += NV * GMS_RED_STRIDE;
        if (++pend == 3) flush(part, lane);
    }
    __device__ __forceinline__ void flush(float (*part)[12], int lane) {
        float* const lcol = col - pend * NV * GMS_RED_STRIDE;      // panel + lane
        gms_red_flush(lcol - lane, part, pj, pend * NV, lane, sh3 - 8 * (3 - pend), ri);
        pend = 0; pj = 0; col = lcol;
    }
};

// Per-lane state of the backward recurrence for the lane's two pixels (index k: row py0 + k).
struct GmsBwdPix {
    float T[2];                // transmittance in front of the current splat, starting from the forward's final T
    float nTbg[2];             // -final T * (bg . dL/dC): the background's share of dL/dalpha is nTbg / (1 - alpha)
    float dpr[2], dpg[2], dpb[2], dpd[2];   // dL/dC, dL/d(inverse depth)
    float Bdot[2];             // (colour, inverse depth) behind the current splat . (dL/dC, dL/dD)
    float npy[2];              // -pixel row
    float npx;                 // -pixel column
    int last[2];               // n_contrib
};

__device__ __forceinline__ GmsBwdPix gms_bwd_pix(const GmsTileGeom& g, int W, int H, const float* __restrict__ bg,
                                                 const float* __restrict__ final_T, const int* __restrict__ n_contrib,
                                                 const float* __restrict__ dL_dpix, const float* __restrict__ dL_dinv) {
    GmsBwdPix P;
    const size_t HW = (size_t)H * W;
    const bool in[2] = {g.in0, g.in1};
    P.npx = -(float)g.px;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        float tf = 1.f, r = 0.f, gg = 0.f, b = 0.f, dd = 0.f;
        int la = 0;
        if (in[k]) {
            const size_t pix = (size_t)(g.py0 + k) * W + g.px;
            tf = final_T[pix]; la = n_contrib[pix];
            r = dL_dpix[pix]; gg = dL_dpix[HW + pix]; b = dL_dpix[2 * HW + pix];
            dd = dL_dinv ? dL_dinv[pix] : 0.f;
        }
        P.T[k] = tf;
        P.nTbg[k] = -tf * (bg[0] * r + bg[1] * gg + bg[2] * b);
        P.dpr[k] = r; P.dpg[k] = gg; P.dpb[k] = b; P.dpd[k] = dd;
        P.Bdot[k] = 0.f;
        P.npy[k] = -(float)(g.py0 + k);
        P.last[k] = la;
    }
    return P;
}

// One (quad, splat) pair, splat (A, B, C) from the slab at list position `pos`.  Writes the lane's NV moment sums to
// col[i * GMS_RED_STRIDE] and returns true; with CULL, returns false (state untouched) when no pixel of the warp blends it.
// The power / alpha / validity sequence is the forward's (gms_power, gms_exp_fast) operation for operation, so a pixel blends
// here exactly when it blended in the forward pass -- the survivor lists and n_contrib depend on it.
template <bool DEPTH, bool CULL>
__device__ __forceinline__ bool gms_bwd_pair(GmsBwdPix& P, const float4& A, const float4& B, const float2& C, int pos, float* col) {
    const float dx = __fadd_rn(A.x, P.npx);
    const float m2 = __fmul_rn(__fmul_rn(A.z, dx), dx);
    const float nm4 = __fmul_rn(A.w, dx);                   // -(cony*dx): the sign flip is exact
    float dy[2], G[2], al[2];
    bool v[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        dy[k] = __fadd_rn(A.y, P.npy[k]);
        const float power = __fmaf_rn(nm4, dy[k], __fmul_rn(__fmaf_rn(__fmul_rn(B.x, dy[k]), dy[k], m2), -0.5f));
        G[k] = gms_ex2(__fmul_rn(power, GMS_LOG2E));
        const float a = fminf(GMS_ALPHA_MAX, __fmul_rn(B.y, G[k]));
        v[k] = pos < P.last[k] && power <= 0.0f && a >= GMS_ALPHA_MIN;
        al[k] = v[k] ? a : 0.f;
    }
    if (CULL && !__any_sync(0xffffffffu, v[0] || v[1])) return false;
    float q[2], w[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const float oma = __fsub_rn(1.f, al[k]);
        const float inv = gms_rcp(oma);
        P.T[k] = __fmul_rn(P.T[k], inv);
        w[k] = __fmul_rn(al[k], P.T[k]);
        float cdp = __fmaf_rn(B.w, P.dpg[k], __fmul_rn(B.z, P.dpr[k]));     // c . dL/dC of this splat
        cdp = __fmaf_rn(C.x, P.dpb[k], cdp);
        if (DEPTH) cdp = __fmaf_rn(C.y, P.dpd[k], cdp);
        // dL/dalpha = (c - B) . dL/dC * T  + background term;  then B <- alpha*c + (1-alpha)*B
        const float dLa = __fmaf_rn(P.nTbg[k], inv, __fmul_rn(__fsub_rn(cdp, P.Bdot[k]), P.T[k]));
        P.Bdot[k] = __fmaf_rn(al[k], cdp, __fmul_rn(oma, P.Bdot[k]));
        q[k] = v[k] ? __fmul_rn(dLa, G[k]) : 0.f;
    }
    // moments: both pixels share dx, so sum q dx^n = dx^n * sum q and sum q dx dy = dx * sum q dy
    const float qy0 = __fmul_rn(q[0], dy[0]), qy1 = __fmul_rn(q[1], dy[1]);
    const float sq = __fadd_rn(q[0], q[1]), sqy = __fadd_rn(qy0, qy1);
    const float sqx = __fmul_rn(dx, sq);
    col[0 * GMS_RED_STRIDE] = sqx;
    col[1 * GMS_RED_STRIDE] = sqy;
    col[2 * GMS_RED_STRIDE] = __fmul_rn(dx, sqx);
    col[3 * GMS_RED_STRIDE] = __fmul_rn(dx, sqy);
    col[4 * GMS_RED_STRIDE] = __fmaf_rn(qy1, dy[1], __fmul_rn(qy0, dy[0]));
    col[5 * GMS_RED_STRIDE] = sq;
    col[6 * GMS_RED_STRIDE] = __fmaf_rn(w[1], P.dpr[1], __fmul_rn(w[0], P.dpr[0]));
    col[7 * GMS_RED_STRIDE] = __fmaf_rn(w[1], P.dpg[1], __fmul_rn(w[0], P.dpg[0]));
    col[8 * GMS_RED_STRIDE] = __fmaf_rn(w[1], P.dpb[1], __fmul_rn(w[0], P.dpb[0]));
    if (DEPTH) col[9 * GMS_RED_STRIDE] = __fmaf_rn(w[1], P.dpd[1], __fmul_rn(w[0], P.dpd[0]));
    return true;
}

// Per-splat epilogue of a round: the splat of slab slot `lane` turns its warp-reduced sums into the gradient record.
template <bool DEPTH>
__device__ __forceinline__ void gms_bwd_commit(const GmsSlabB& S, int lane, float halfW, float halfH, float4* __restrict__ dgeom) {
    const int id = S.id[lane];
    const float4 s0 = *reinterpret_cast<const float4*>(&S.part[lane][0]);
    const float4 s1 = *reinterpret_cast<const float4*>(&S.part[lane][4]);
    float2 s2 = *reinterpret_cast<const float2*>(&S.part[lane][8]);
    if (!DEPTH) s2.y = 0.f;                 // the 9-value panel never writes the inverse-depth sum
    const float4 A = S.a[lane];
    const float2 B = make_float2(S.b[lane].x, S.b[lane].y);
    const float conx = A.z, ncony = A.w, conz = B.x, op = B.y;
    float4 g0, g1;
    g0.x = (-conx * s0.x + ncony * s0.y) * op * halfW;  // dL/dmean2D.x (NDC-scaled)
    g0.y = (-conz * s0.y + ncony * s0.x) * op * halfH;  // dL/dmean2D.y
    g0.z = -0.5f * op * s0.z;                           // dL/dconic.x
    g0.w = -0.5f * op * s0.w;                           // dL/dconic.y (stock half convention)
    g1.x = -0.5f * op * s1.x;                           // dL/dconic.z
    g1.y = s1.y;                                        // dL/d(conic_opacity.w)
    g1.z = s1.z; g1.w = s1.w;                           // dL/drgb.r, .g
    atomicAdd(&dgeom[3 * id], g0);
    atomicAdd(&dgeom[3 * id + 1], g1);
    atomicAdd(reinterpret_cast<float2*>(&dgeom[3 * id + 2]), s2);   // dL/drgb.b, dL/dinvdepth
}

// DEPTH = false: no loss on the inverse-depth image (train.py never puts one): the depth channel of the recurrence and its
// moment sum are compiled out.  The panel holds exactly 3*NV rows: 27 KB of shared memory per CTA without DEPTH, which
// leaves room for 8 CTAs per SM.
template <int MINB, bool DEPTH>
__global__ void __launch_bounds__(GMS_CB, MINB)
k_composite_bwd5(const int2* __restrict__ ranges, const int* __restrict__ tile_order, const uint32_t* __restrict__ point_list,
                 const float4* __restrict__ recs, int W, int H, int gx, const float* __restrict__ bg,
                 const float* __restrict__ final_T, const int* __restrict__ n_contrib,
                 const float* __restrict__ dL_dpix, const float* __restrict__ dL_dinv, float4* __restrict__ dgeom,
                 const uint32_t* __restrict__ surv, const uint32_t* __restrict__ nsurv) {
    constexpr int NV = DEPTH ? 10 : 9;         // partial sums per splat
    __shared__ GmsSlabB s_slab[4];
    __shared__ __align__(16) float s_red[4][3 * NV * GMS_RED_STRIDE];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = tile_order ? tile_order[blockIdx.x] : (int)blockIdx.x;
    const GmsTileGeom g = gms_tile_geom(tile, gx, W, H, warp, lane);
    const int2 rng = ranges[tile];
    const float halfW = 0.5f * (float)W, halfH = 0.5f * (float)H;
    GmsSlabB& S = s_slab[warp];
    GmsPanel<NV> R(s_red[warp], lane);
    const int cnt = (int)nsurv[4 * tile + warp];          // (quad, splat) pairs that blended in the forward pass
    if (cnt <= 0) return;
    const uint32_t* __restrict__ ql = surv + 4 * (size_t)rng.x + (size_t)warp * (rng.y - rng.x);
    const uint32_t* __restrict__ plist = point_list + rng.x;
    GmsBwdPix P = gms_bwd_pix(g, W, H, bg, final_T, n_contrib, dL_dpix, dL_dinv);
    const int nb = (cnt + GMS_WB - 1) / GMS_WB;

    // software pipeline: positions + ids two rounds ahead, records one round ahead
    int pos_cur = -1, id_cur = -1, pos_nx = -1, id_nx = -1;
    float4 ra = make_float4(0, 0, 0, 0), rb = ra, rc = ra;
    {
        const int k = (nb - 1) * GMS_WB + lane;
        if (k < cnt) { pos_cur = (int)ql[k]; id_cur = (int)plist[pos_cur]; ra = recs[3 * id_cur]; rb = recs[3 * id_cur + 1]; rc = recs[3 * id_cur + 2]; }
        if (nb >= 2) { pos_nx = (int)ql[(nb - 2) * GMS_WB + lane]; id_nx = (int)plist[pos_nx]; }
    }
    for (int b = nb - 1; b >= 0; b--) {
        S.id[lane] = id_cur; S.pos[lane] = pos_cur;
        if (id_cur >= 0) gms_slabb_store(S, lane, ra, rb, rc);
        uint32_t m = __ballot_sync(0xffffffffu, id_cur >= 0);
        const uint32_t touched = m;
        id_cur = id_nx; pos_cur = pos_nx;
        if (id_cur >= 0) { ra = recs[3 * id_cur]; rb = recs[3 * id_cur + 1]; rc = recs[3 * id_cur + 2]; }
        if (b >= 2) { pos_nx = (int)ql[(b - 2) * GMS_WB + lane]; id_nx = (int)plist[pos_nx]; } else { pos_nx = -1; id_nx = -1; }
        __syncwarp();
        while (m) {
            const int j = 31 - __clz(m);
            m ^= 1u << j;
            gms_bwd_pair<DEPTH, false>(P, S.a[j], S.b[j], S.c[j], S.pos[j], R.col);
            R.push(j, S.part, lane);
        }
        if (R.pend) R.flush(S.part, lane);
        __syncwarp();
        if ((touched >> lane) & 1u) gms_bwd_commit<DEPTH>(S, lane, halfW, halfH, dgeom);
        __syncwarp();
    }
}

// Predecessor: streams the tile's whole list and culls per quad (ellipse vs rectangle), then the same per-pair step.
template <int MINB, bool DEPTH>
__global__ void __launch_bounds__(GMS_CB, MINB)
k_composite_bwd3(const int2* __restrict__ ranges, const int* __restrict__ tile_order, const uint32_t* __restrict__ point_list,
                 const float4* __restrict__ recs, int W, int H, int gx, const float* __restrict__ bg,
                 const float* __restrict__ final_T, const int* __restrict__ n_contrib,
                 const float* __restrict__ dL_dpix, const float* __restrict__ dL_dinv, float4* __restrict__ dgeom) {
    constexpr int NV = DEPTH ? 10 : 9;         // partial sums per splat
    __shared__ GmsSlabB s_slab[4];
    __shared__ __align__(16) float s_red[4][3 * NV * GMS_RED_STRIDE];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = tile_order ? tile_order[blockIdx.x] : (int)blockIdx.x;
    const GmsTileGeom g = gms_tile_geom(tile, gx, W, H, warp, lane);
    const int2 rng = ranges[tile];
    const float halfW = 0.5f * (float)W, halfH = 0.5f * (float)H;
    GmsSlabB& S = s_slab[warp];
    GmsPanel<NV> R(s_red[warp], lane);
    const float qx0 = (float)(g.tx0 + (warp & 1) * 8), qy0 = (float)(g.ty0 + (warp >> 1) * 8);
    GmsBwdPix P = gms_bwd_pix(g, W, H, bg, final_T, n_contrib, dL_dpix, dL_dinv);
    const int wlast = __reduce_max_sync(0xffffffffu, max(P.last[0], P.last[1]));
    if (wlast <= 0) return;
    const int nb = (wlast + GMS_WB - 1) / GMS_WB;

    int id_cur;
    float4 ra = make_float4(0, 0, 0, 0), rb = ra, rc = ra;
    {
        const int k = (nb - 1) * GMS_WB + lane;
        id_cur = (k < wlast) ? (int)point_list[rng.x + k] : -1;
        if (id_cur >= 0) { ra = recs[3 * id_cur]; rb = recs[3 * id_cur + 1]; rc = recs[3 * id_cur + 2]; }
    }
    int id_nx = (nb >= 2) ? (int)point_list[rng.x + (nb - 2) * GMS_WB + lane] : -1;

    for (int b = nb - 1; b >= 0; b--) {
        bool hit = false;
        S.id[lane] = id_cur;
        if (id_cur >= 0) {
            hit = gms_reaches_quad(ra.x, ra.y, ra.z, ra.w, rb.x, rc.z, qx0, qy0);
            if (hit) gms_slabb_store(S, lane, ra, rb, rc);
        }
        uint32_t m = __ballot_sync(0xffffffffu, hit);
        id_cur = id_nx;
        if (id_cur >= 0) { ra = recs[3 * id_cur]; rb = recs[3 * id_cur + 1]; rc = recs[3 * id_cur + 2]; }
        id_nx = (b >= 2) ? (int)point_list[rng.x + (b - 2) * GMS_WB + lane] : -1;
        __syncwarp();
        uint32_t touched = 0;
        while (m) {
            const int j = 31 - __clz(m);
            m ^= 1u << j;
            if (!gms_bwd_pair<DEPTH, true>(P, S.a[j], S.b[j], S.c[j], b * GMS_WB + j, R.col)) continue;
            R.push(j, S.part, lane);
            touched |= 1u << j;
        }
        if (R.pend) R.flush(S.part, lane);
        __syncwarp();
        if ((touched >> lane) & 1u) gms_bwd_commit<DEPTH>(S, lane, halfW, halfH, dgeom);
        __syncwarp();
    }
}
