// gms_composite_common.cuh -- shared pieces of the per-tile compositing kernels, sm_90a.
//
// Replaces (together with gms_composite_fwd.cuh / gms_composite_bwd.cuh) [upstream forward.cu: renderCUDA] and
// [upstream backward.cu: renderCUDA] of graphdeco-inria/diff-gaussian-rasterization (reference call sites:
// renderer/gaussian_renderer/__init__.py:94-102, train.py:108).  Semantics: SURVEY.md Appendix A.2 / A.3, checked by the
// CPU oracle under oracle/.
//
// Work decomposition (differs from the stock one-thread-per-pixel / per-pixel-atomics kernels):
//  * a 16x16 tile is owned by a 128-thread CTA; each warp owns an 8x8 pixel QUAD, each lane two vertically adjacent
//    pixels (the x-dependent half of the quadratic form is shared between them, ILP = 2);
//  * every warp streams the tile's depth-sorted list ON ITS OWN, 32 splats per round, through a warp-private
//    shared-memory slab -- no block-level barrier anywhere in the loop, a warp whose 64 pixels are saturated exits;
//  * an exact ellipse-vs-rectangle test decides which staged splats can reach the warp's quad at alpha >= 1/255;
//  * tiles are launched longest list first (k_tile_order).
// Superseded generations (block-synchronous batches, shuffle-fold backward, octet lists) live in
// experiments/composite_generations/ with their measurements; they are not part of the library.
#pragma once
#include "gms_common.cuh"

#define GMS_CB 128                  // CTA size: four warps = four 8x8 quads
#define GMS_WB 32                   // splats staged per warp round
#define GMS_LOG2E 1.4426950408889634f

// canonical quadratic form (see oracle quad_power): shared x-part
__device__ __forceinline__ float gms_power(float m2, float m4, float conz, float dy) {
    const float m3 = __fmul_rn(conz, dy);
    const float t = __fmaf_rn(m3, dy, m2);
    const float h = __fmul_rn(-0.5f, t);
    return __fmaf_rn(-m4, dy, h);
}

struct GmsTileGeom {
    int tx0, ty0, px, py0;
    bool in0, in1;
};

__device__ __forceinline__ GmsTileGeom gms_tile_geom(int tile, int gx, int W, int H, int warp, int lane) {
    GmsTileGeom g;
    g.tx0 = (tile % gx) * GMS_TILE;
    g.ty0 = (tile / gx) * GMS_TILE;
    g.px = g.tx0 + (warp & 1) * 8 + (lane & 7);
    g.py0 = g.ty0 + (warp >> 1) * 8 + (lane >> 3) * 2;
    g.in0 = g.px < W && g.py0 < H;
    g.in1 = g.px < W && (g.py0 + 1) < H;
    return g;
}

// Can this splat reach alpha >= 1/255 anywhere in the pixel rectangle [rx0, rx0+7] x [ry0, ry0+7]?
// i.e. min over the rectangle of 0.5*(cx dx^2 + cz dy^2) + cy dx dy  <=  tau   (tau carries the safety margin).
__device__ __forceinline__ bool gms_reaches_quad(float x, float y, float cx, float cy, float cz, float tau, float rx0, float ry0) {
    if (!(tau > 0.f)) return false;                 // opacity < 1/255: never blends
    if (!(cx > 0.f) || !(cz > 0.f)) return true;    // degenerate conic: be conservative
    const float rx1 = rx0 + 7.0f, ry1 = ry0 + 7.0f;
    if (x >= rx0 && x <= rx1 && y >= ry0 && y <= ry1) return true;
    float best = 3.0e38f;
    const float icx = __fdividef(1.f, cx), icz = __fdividef(1.f, cz);
#pragma unroll
    for (int e = 0; e < 2; e++) {
        {   // horizontal edge
            const float dy = y - (e ? ry1 : ry0);
            const float t = fminf(fmaxf(x + cy * dy * icx, rx0), rx1);
            const float dx = x - t;
            best = fminf(best, 0.5f * (cx * dx * dx + cz * dy * dy) + cy * dx * dy);
        }
        {   // vertical edge
            const float dx = x - (e ? rx1 : rx0);
            const float t = fminf(fmaxf(y + cy * dx * icz, ry0), ry1);
            const float dy = y - t;
            best = fminf(best, 0.5f * (cx * dx * dx + cz * dy * dy) + cy * dx * dy);
        }
    }
    return best <= tau;
}

__device__ __forceinline__ float gms_exp_fast(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(__fmul_rn(x, GMS_LOG2E)));
    return y;
}

struct GmsWarpSlab {          // one per warp, two for the forward's double buffering
    float4 a[GMS_WB];         // x, y, conx, cony
    float4 b[GMS_WB];         // conz, opacity, r, g
    float2 c[GMS_WB];         // b, 1/depth
};

// ------------------------------------------------------------------------------------------- tile order
// Longest list first: counting sort of the T tiles into 33 buckets by bit-length of their list (one CTA).  Most tiles fall into
// four or five buckets, so the shared-memory atomics are aggregated per warp: lanes with the same bucket elect a leader that
// adds their count once (match.any), the others take their rank from the peer mask.
__global__ void __launch_bounds__(1024) k_tile_order(int T, const int2* __restrict__ ranges, int* __restrict__ order) {
    __shared__ int s_cnt[33];
    __shared__ int s_off[33];
    const int lane = threadIdx.x & 31;
    if (threadIdx.x < 33) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const int n = ranges[t].y - ranges[t].x;
        const int b = n > 0 ? 32 - __clz(n) : 0;
        const unsigned peers = __match_any_sync(__activemask(), b);
        if (lane == __ffs(peers) - 1) atomicAdd(&s_cnt[b], __popc(peers));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int b = 32; b >= 0; b--) { s_off[b] = run; run += s_cnt[b]; }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const int n = ranges[t].y - ranges[t].x;
        const int b = n > 0 ? 32 - __clz(n) : 0;
        const unsigned peers = __match_any_sync(__activemask(), b);
        const int leader = __ffs(peers) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(&s_off[b], __popc(peers));
        base = __shfl_sync(peers, base, leader);
        order[base + __popc(peers & ((1u << lane) - 1u))] = t;
    }
}

typedef float2 f2;

// Two-lane float arithmetic.  sm_90 has no packed f32x2 FMA pipe, so each lane is one scalar round-to-nearest FFMA / FMUL /
// FADD; the explicit intrinsics keep nvcc from contracting a mul + add into an FMA, so results are bit-identical to the
// scalar kernels.
__device__ __forceinline__ f2 f2fma(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 f2mul(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2 f2add(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float gms_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float gms_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct GmsSlab3 {              // pair-duplicated per-splat data of the float2-pair forward (k_composite_fwd3)
    float4 q0[GMS_WB];         // x, x, y, y
    float4 q1[GMS_WB];         // conx, conx, -cony, -cony
    float4 q2[GMS_WB];         // conz, conz, op, op
    float4 q3[GMS_WB];         // r, r, g, g
    float4 q4[GMS_WB];         // b, b, invd, invd
};

__device__ __forceinline__ void gms_slab3_store(GmsSlab3& S, int lane, const float4& ra, const float4& rb, const float4& rc) {
    S.q0[lane] = make_float4(ra.x, ra.x, ra.y, ra.y);
    S.q1[lane] = make_float4(ra.z, ra.z, -ra.w, -ra.w);
    S.q2[lane] = make_float4(rb.x, rb.x, rb.y, rb.y);
    S.q3[lane] = make_float4(rb.z, rb.z, rb.w, rb.w);
    S.q4[lane] = make_float4(rc.x, rc.x, rc.y, rc.y);
}

// canonical quadratic form for the pixel pair: power = fma(-(cy*dx), dy, -0.5 * fma(cz*dy, dy, (cx*dx)*dx))
__device__ __forceinline__ f2 gms_power2(const float4& Q0, const float4& Q1, const float4& Q2, f2 npx, f2 npy, f2& dx, f2& dy) {
    dx = f2add(make_float2(Q0.x, Q0.y), npx);
    dy = f2add(make_float2(Q0.z, Q0.w), npy);
    const f2 m1 = f2mul(make_float2(Q1.x, Q1.y), dx);
    const f2 m2 = f2mul(m1, dx);
    const f2 nm4 = f2mul(make_float2(Q1.z, Q1.w), dx);          // -(cony*dx): the sign flip is exact
    const f2 m3 = f2mul(make_float2(Q2.x, Q2.y), dy);
    const f2 t = f2fma(m3, dy, m2);
    const f2 h = f2mul(t, make_float2(-0.5f, -0.5f));
    return f2fma(nm4, dy, h);
}

