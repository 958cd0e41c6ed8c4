// gms_raster.cuh -- the rasterizer's per-Gaussian kernels around binning and compositing, sm_90a: the preprocess
// forward and backward (SH rows staged through shared memory, the fused SH Adam step), duplicate emission, tile ranges,
// the background fill, and the debug / visibility helpers.  The maths they call is in gms_preprocess.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "gms_common.cuh"
#include "gms_preprocess.cuh"
#include "gms_adam.cuh"

struct PreArgs {
    int P, D, M, W, H, gx, gy, antialiasing;
    float tanfovx, tanfovy, focal_x, focal_y, mod;
    const float* means; const float* scales; const float* rots; const float* cov_pre; const float* opac;
    const float* opac_raw; float* opac_out;     // gms_train_frame: opacity = sigmoid(opac_raw), computed here and stored to opac_out (= opac for the backward)
    const float* shs; const float* colors_pre;
    const float* view; const float* proj; const float* campos;
};

// SH rows (M = 16: 48 floats = 192 B per Gaussian) are 192 B apart between lanes: read directly, every 128-bit load of a
// warp touches 32 different sectors.  STAGED: the warp's 32 rows are one contiguous 6 KB block, copied with fully
// coalesced 128-bit accesses into (out of) a padded shared-memory tile, row stride 13 float4 = conflict-free for both
// the cooperative and the per-lane pattern.  Rows of culled Gaussians are skipped on load and written as zeros on store.
constexpr int GMS_SH_ROW4 = 12;
constexpr int GMS_SH_STRIDE_V = 52;    // floats per tile row, 128-bit per-lane accesses (13 float4: conflict-free)
constexpr int GMS_SH_STRIDE_S = 49;    // floats per tile row, scalar per-lane accesses (odd: conflict-free)
constexpr int GMS_SH_TILE = 32 * GMS_SH_STRIDE_V;      // floats of shared memory per warp (either layout fits)

// NC: through the read-only data cache.  Not when the same kernel later writes the rows (the fused SH Adam update).
template <int STRIDE, bool NC = true>
__device__ __forceinline__ void sh_tile_load(const float* shs, int i0, unsigned rows, int lane, float* t) {
    const float4* src = reinterpret_cast<const float4*>(shs) + (size_t)i0 * GMS_SH_ROW4;
#pragma unroll
    for (int it = 0; it < GMS_SH_ROW4; it++) {
        const int j = it * 32 + lane, r = j / GMS_SH_ROW4, c = j - r * GMS_SH_ROW4;
        if ((rows >> r) & 1u) {
            const float4 v = NC ? __ldg(src + j) : src[j];
            float* d = t + r * STRIDE + 4 * c;
            if (STRIDE % 4 == 0) *reinterpret_cast<float4*>(d) = v;
            else { d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w; }
        }
    }
    __syncwarp();
}
template <int STRIDE>
__device__ __forceinline__ void sh_tile_store(float* __restrict__ dshs, int i0, int P, int lane, const float* t) {
    __syncwarp();
    float4* dst = reinterpret_cast<float4*>(dshs) + (size_t)i0 * GMS_SH_ROW4;
#pragma unroll
    for (int it = 0; it < GMS_SH_ROW4; it++) {
        const int j = it * 32 + lane, r = j / GMS_SH_ROW4, c = j - r * GMS_SH_ROW4;
        if (i0 + r < P) {
            const float* q = t + r * STRIDE + 4 * c;
            dst[j] = (STRIDE % 4 == 0) ? *reinterpret_cast<const float4*>(q) : make_float4(q[0], q[1], q[2], q[3]);
        }
    }
}

template <bool STAGED>
__global__ void __launch_bounds__(128)
k_preprocess_fwd(PreArgs a, int* __restrict__ radii, float4* __restrict__ rec, float* __restrict__ cov3D,
                 uint32_t* __restrict__ clamped, uint32_t* __restrict__ tiles, uint32_t* __restrict__ dkey,
                 uint32_t* __restrict__ idx, uint2* __restrict__ rect, uint32_t* __restrict__ counters) {
    __shared__ __align__(16) float s_sh[STAGED ? 4 : 1][STAGED ? GMS_SH_TILE : 4];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (!STAGED && i >= a.P) return;
    const bool inb = i < a.P;
    GmsPre o;
    bool vis = false;
    float mean[3] = {0.f, 0.f, 0.f};
    if (inb) {
        float view[16], proj[16];
#pragma unroll
        for (int k = 0; k < 16; k++) { view[k] = __ldg(a.view + k); proj[k] = __ldg(a.proj + k); }
        mean[0] = a.means[3 * i]; mean[1] = a.means[3 * i + 1]; mean[2] = a.means[3 * i + 2];
        float sc[3] = {0, 0, 0}, rt[4] = {1, 0, 0, 0}, cv[6];
        const float* cvp = nullptr;
        if (a.cov_pre) {
#pragma unroll
            for (int k = 0; k < 6; k++) cv[k] = a.cov_pre[6 * (size_t)i + k];
            cvp = cv;
        } else {
            sc[0] = a.scales[3 * i]; sc[1] = a.scales[3 * i + 1]; sc[2] = a.scales[3 * i + 2];
            const float4 q = reinterpret_cast<const float4*>(a.rots)[i];
            rt[0] = q.x; rt[1] = q.y; rt[2] = q.z; rt[3] = q.w;
        }
        float opacity;
        if (a.opac_raw) { opacity = GMS_DIVP(1.0f, 1.0f + expf(-a.opac_raw[i])); a.opac_out[i] = opacity; }    // scene/gaussian_model.py:113-115 (sigmoid), fused
        else opacity = a.opac[i];
        vis = gms_preprocess_geom(mean, sc, rt, cvp, opacity, view, proj, a.W, a.H, a.tanfovx, a.tanfovy,
                                  a.focal_x, a.focal_y, a.mod, a.antialiasing, a.gx, a.gy, o);
        idx[i] = (uint32_t)i;
        if (!vis) { radii[i] = 0; tiles[i] = 0; dkey[i] = 0xFFFFFFFFu; rect[i] = make_uint2(0u, 0u); }
        else rect[i] = make_uint2((uint32_t)o.x0 | ((uint32_t)o.y0 << 16), (uint32_t)o.x1 | ((uint32_t)o.y1 << 16));
    }
    if (STAGED) {       // (only launched with shs != NULL and M == 16; no thread has left: full-warp votes)
        const unsigned rows = __ballot_sync(0xffffffffu, vis);
        // visible Gaussians / sum of tiles_touched of this CTA: one pair of global atomics per CTA
        __shared__ uint32_t s_cnt[4][2];
        const uint32_t wt = __reduce_add_sync(0xffffffffu, vis ? o.tiles : 0u);
        if (lane == 0) { s_cnt[warp][0] = (uint32_t)__popc(rows); s_cnt[warp][1] = wt; }
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t nv = s_cnt[0][0] + s_cnt[1][0] + s_cnt[2][0] + s_cnt[3][0];
            if (nv) { atomicAdd(counters + 2, nv); atomicAdd(counters + 3, s_cnt[0][1] + s_cnt[1][1] + s_cnt[2][1] + s_cnt[3][1]); }
        }
        if (rows) sh_tile_load<GMS_SH_STRIDE_V>(a.shs, blockIdx.x * blockDim.x + warp * 32, rows, lane, s_sh[warp]);
    }
    if (!STAGED && vis) { atomicAdd(counters + 2, 1u); atomicAdd(counters + 3, o.tiles); }
    if (!vis) return;
    float rgb[3];
    uint8_t cl[3] = {0, 0, 0};
    if (a.shs) {
        float sh[48];
        const int nf = 3 * (a.D + 1) * (a.D + 1);
        if (STAGED) {
#pragma unroll
            for (int k = 0; k < 12; k++) {
                if (4 * k < nf) {
                    const float4 v = *reinterpret_cast<const float4*>(&s_sh[warp][lane * GMS_SH_STRIDE_V + 4 * k]);
                    sh[4 * k] = v.x; sh[4 * k + 1] = v.y; sh[4 * k + 2] = v.z; sh[4 * k + 3] = v.w;
                }
            }
        } else {
            const float* row = a.shs + (size_t)i * a.M * 3;
            if (((a.M * 3) & 3) == 0) {
                const float4* r4 = reinterpret_cast<const float4*>(row);
#pragma unroll
                for (int k = 0; k < 12; k++) {
                    if (4 * k < nf) {
                        const float4 v = __ldg(r4 + k);
                        sh[4 * k] = v.x; sh[4 * k + 1] = v.y; sh[4 * k + 2] = v.z; sh[4 * k + 3] = v.w;
                    }
                }
            } else {
#pragma unroll
                for (int k = 0; k < 48; k++) if (k < nf) sh[k] = __ldg(row + k);
            }
        }
        const float campos[3] = {__ldg(a.campos), __ldg(a.campos + 1), __ldg(a.campos + 2)};
        gms_sh_color(a.D, mean, campos, sh, rgb, cl);
    } else {
        rgb[0] = a.colors_pre[3 * i]; rgb[1] = a.colors_pre[3 * i + 1]; rgb[2] = a.colors_pre[3 * i + 2];
    }
    // tau' = ln(255 * opacity) + margin: a pixel can blend (alpha >= 1/255) only where 0.5 d^T Q d <= tau'.  The composite
    // kernels test each tile quad against that ellipse before visiting the splat (gms_reaches_quad).  Margin (DESIGN.md 3.4):
    // 1% + 1e-3 for ex2.approx and logf; 1e-3 * (|cx| + |cz| + 2|cy|) for the rounding of the per-pixel power across the
    // 7 x 7 px of a quad and for the cull's own edge minimiser.  The part that grows with the magnitude of the quadratic form's
    // terms (edge-on slivers: up to ~1e9) is subtracted inside the cull, point by point.
    const float tau = (o.opac >= GMS_ALPHA_MIN)
        ? 1.01f * logf(255.0f * o.opac) + 1e-3f * (1.0f + fabsf(o.conx) + fabsf(o.conz) + 2.0f * fabsf(o.cony)) : -1.0f;
    rec[3 * (size_t)i] = make_float4(o.px, o.py, o.conx, o.cony);
    rec[3 * (size_t)i + 1] = make_float4(o.conz, o.opac, rgb[0], rgb[1]);
    rec[3 * (size_t)i + 2] = make_float4(rgb[2], GMS_DIVP(1.f, o.depth), tau, 0.f);
    float2* c2 = reinterpret_cast<float2*>(cov3D + 6 * (size_t)i);
    c2[0] = make_float2(o.cov6[0], o.cov6[1]); c2[1] = make_float2(o.cov6[2], o.cov6[3]); c2[2] = make_float2(o.cov6[4], o.cov6[5]);
    clamped[i] = (uint32_t)cl[0] | ((uint32_t)cl[1] << 1) | ((uint32_t)cl[2] << 2);
    radii[i] = o.radius;
    tiles[i] = o.tiles;
    dkey[i] = __float_as_uint(o.depth);
}

// one thread (small rect) or one warp (large rect) per Gaussian, in depth order
// KeyT: uint16_t when the tile count fits (T <= 65535: 16 B instead of 20 B per duplicate through the tile sort), else uint32_t.
template <typename KeyT>
__global__ void __launch_bounds__(256)
k_emit_dups(int P, int gx, const uint32_t* __restrict__ order, const uint32_t* __restrict__ offs, const uint2* __restrict__ rect,
            KeyT* __restrict__ keys, uint32_t* __restrict__ vals, int warp_coop, uint32_t cap) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t g = 0, nt = 0, off = 0;
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (j < P) {
        g = order[j];
        const uint2 r = rect[g];            // ONE 8-byte gather per Gaussian: the packed tile rectangle k_preprocess_fwd wrote
        x0 = (int)(r.x & 0xFFFFu); y0 = (int)(r.x >> 16); x1 = (int)(r.y & 0xFFFFu); y1 = (int)(r.y >> 16);
        nt = (uint32_t)((x1 - x0) * (y1 - y0));
        if (nt) off = j ? offs[j - 1] : 0u;
    }
    const uint32_t big_thresh = 32;
    const bool big = warp_coop && nt >= big_thresh;
    if (nt && !big) {
        for (int y = y0; y < y1; y++)
            for (int x = x0; x < x1; x++) {
                if (off < cap) { keys[off] = (KeyT)(y * gx + x); vals[off] = g; }     // (cap < N: overflow frame, flagged by k_tile_ranges)
                off++;
            }
    }
    uint32_t bigmask = __ballot_sync(0xffffffffu, big);
    while (bigmask) {
        const int src = __ffs(bigmask) - 1;
        bigmask &= bigmask - 1;
        const uint32_t g_s = __shfl_sync(0xffffffffu, g, src);
        const uint32_t nt_s = __shfl_sync(0xffffffffu, nt, src);
        const uint32_t off_s = __shfl_sync(0xffffffffu, off, src);
        const int x0_s = __shfl_sync(0xffffffffu, x0, src), y0_s = __shfl_sync(0xffffffffu, y0, src);
        const int w_s = __shfl_sync(0xffffffffu, x1, src) - x0_s;
        for (uint32_t k = lane; k < nt_s; k += 32) {
            const int yy = y0_s + (int)(k / (uint32_t)w_s), xx = x0_s + (int)(k % (uint32_t)w_s);
            if (off_s + k < cap) { keys[off_s + k] = (KeyT)(yy * gx + xx); vals[off_s + k] = g_s; }
        }
    }
}

// `cap` sorted entries of which the first N (device) are real; the tail holds sentinel keys (>= T).  N > cap: overflow --
// every range stays (0, 0) (the caller zero-filled them), the flag is raised, the frame renders the background.
template <typename KeyT>
__global__ void __launch_bounds__(256)
k_tile_ranges(int64_t cap, const KeyT* __restrict__ keys, int2* __restrict__ ranges, uint32_t T, const uint32_t* __restrict__ d_n,
              uint32_t* __restrict__ n_out, volatile uint32_t* n_host) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t N = *d_n;
    const bool overflow = (int64_t)N > cap;
    if (j == 0) {
        if (n_out) { n_out[0] = N; n_out[1] = overflow ? 1u : 0u; }
        if (n_host) { n_host[0] = N; n_host[1] = overflow ? 1u : 0u; }
    }
    if (j >= cap || overflow) return;
    const uint32_t t = keys[j];
    if (t >= T) {                                   // sentinel tail
        if (j > 0) { const uint32_t tp = keys[j - 1]; if (tp < T) ranges[tp].y = (int)j; }
        return;
    }
    if (j == 0) ranges[t].x = 0;
    else {
        const uint32_t tp = keys[j - 1];
        if (tp != t) { ranges[tp].y = (int)j; ranges[t].x = (int)j; }
    }
    if (j == cap - 1) ranges[t].y = (int)cap;
}

__global__ void k_fill_background(int W, int H, const float* __restrict__ bg, float* __restrict__ out_color,
                                  float* __restrict__ out_invdepth) {
    const size_t HW = (size_t)W * H;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= HW) return;
    out_color[i] = bg[0]; out_color[HW + i] = bg[1]; out_color[2 * HW + i] = bg[2];
    out_invdepth[i] = 0.f;
}

constexpr int GMS_SH_FSTRIDE = 19;     // floats per lane of the factor tile: 16 basis values + 3 colour gradients (odd: conflict-free)

// The fused update of a warp's 32 rows, after the preprocess backward (every lane of the warp takes part).  tile: the rows
// (p) at row stride GMS_SH_STRIDE_V, loaded for every in-bounds Gaussian.  f: the lane's factors, which k_adam_sh's phase A
// would have multiplied out with one rank and scale 1 -- the basis and the clamp-masked colour gradient, or zeros when the
// whole colour gradient is zero (culled / unblended / clamped).  The walk over p / m / v is k_adam_sh's phase B, with p from
// the tile instead of memory and the gradient formed as the same single product basis_k * dcolor[c].
template <bool IEEE_CALLS>
__device__ __forceinline__ void sh_adam_warp(const AdamShConst& ac, float* p, float* m, float* v, int P, int i0, int lane,
                                             const float* tile, const float* f) {
    const size_t base4 = (size_t)i0 * GMS_SH_ROW4;
    const float4* m4 = reinterpret_cast<const float4*>(m) + base4;
    const float4* v4 = reinterpret_cast<const float4*>(v) + base4;
    const int nrow = min(32, P - i0), n4 = GMS_SH_ROW4 * nrow;
    constexpr int AHEAD = 2;
    float4 Mb[AHEAD + 1], Vb[AHEAD + 1];
#pragma unroll
    for (int q = 0; q < AHEAD; q++) {
        Mb[q] = Vb[q] = make_float4(0, 0, 0, 0);
        if (q * 32 + lane < n4) { Mb[q] = m4[q * 32 + lane]; Vb[q] = v4[q * 32 + lane]; }
    }
    __syncwarp();
    float4* po = reinterpret_cast<float4*>(p) + base4;
    float4* mo = reinterpret_cast<float4*>(m) + base4;
    float4* vo = reinterpret_cast<float4*>(v) + base4;
#pragma unroll
    for (int it = 0; it < GMS_SH_ROW4; it++) {
        const int j = it * 32 + lane;
        if (it + AHEAD < GMS_SH_ROW4) {
            const int jn = j + AHEAD * 32, sl = (it + AHEAD) % (AHEAD + 1);
            Mb[sl] = Vb[sl] = make_float4(0, 0, 0, 0);
            if (jn < n4) { Mb[sl] = m4[jn]; Vb[sl] = v4[jn]; }
        }
        const float4 Mc = Mb[it % (AHEAD + 1)], Vc = Vb[it % (AHEAD + 1)];
        if (j < n4) {
            const int r = j / GMS_SH_ROW4, c = j - r * GMS_SH_ROW4;
            const float4 Pc = *reinterpret_cast<const float4*>(tile + r * GMS_SH_STRIDE_V + 4 * c);
            const float* fr = f + r * GMS_SH_FSTRIDE;
            float gv[4];
#pragma unroll
            for (int k = 0; k < 4; k++) { const int e = 4 * c + k, kk = e / 3; gv[k] = fr[kk] * fr[16 + e - 3 * kk]; }
            float pv[4] = {Pc.x, Pc.y, Pc.z, Pc.w}, mv[4] = {Mc.x, Mc.y, Mc.z, Mc.w}, vv[4] = {Vc.x, Vc.y, Vc.z, Vc.w};
            adam_sh_update4<IEEE_CALLS>(ac, c, gv, pv, mv, vv);
            po[j] = make_float4(pv[0], pv[1], pv[2], pv[3]);
            mo[j] = make_float4(mv[0], mv[1], mv[2], mv[3]);
            vo[j] = make_float4(vv[0], vv[1], vv[2], vv[3]);
        }
    }
}

struct PreBwdArgs {
    PreArgs f;
    const int* radii; const float* cov3D; const uint32_t* clamped; const float4* dgeom;
    float* dmeans3D; float* dmeans2D; float* dopac; float* dshs; float* dcolors_pre; float* dscales; float* drots; float* dcov_pre;
    float* dopac_raw;   // gms_train_frame: dL/d(opacity before the sigmoid) = dL/dopacity * y (1 - y) goes here instead of dopac
    float* dcol_sh;     // [P,3] clamp-masked dL/dcolour of SH-coloured Gaussians (factored SH gradient: dL/dSH[k][c] = basis_k(dir) * this[c]); with it dshs may be NULL
    float* sh_p; float* sh_m; float* sh_v; AdamShConst sh_adam;    // ADAM: the SH parameter (= f.shs, updated in place) and its moments
};

// STAGED 0: per-lane global accesses.  1: SH rows and gradient rows through the warp's shared-memory tile, held in
// registers in between (sh[48], dsh[48]).  2: as 1, but gms_sh_backward works IN PLACE on the lane's tile row (scalar,
// odd row stride): no register copies of the two 48-float rows.
// FACT: factored SH gradient -- the SH rows are read (their view-direction term feeds dL/dmean) but no gradient rows are
// written; the clamp-masked colour gradient (12 B instead of 192 B per Gaussian) goes to b.dcol_sh (gms_adam_sh_factored).
// ADAM (with STAGED 1 and FACT; one camera per step): instead of handing the colour gradient to k_adam_sh, the kernel applies
// the SH Adam step itself to the rows it already holds in its tile (sh_adam_warp), so p is not read twice and the exchange
// slot is not needed (b.dcol_sh is then optional).  The tile holds every in-bounds row: culled Gaussians get an update with a
// zero gradient.  p is the SH input itself (b.sh_p == f.shs): each warp reads its rows before it writes them, and no other
// warp touches them, so the rows are loaded without the read-only cache.  ADAM_IEEE: the adam_sh_ieee arm of the update.
template <int STAGED, int MINB, bool FACT = false, bool ADAM = false, bool ADAM_IEEE = false>
__global__ void __launch_bounds__(128, MINB) k_preprocess_bwd(PreBwdArgs b) {
    static_assert(!ADAM || (STAGED == 1 && FACT), "the fused SH Adam update works on the STAGED 1 tile of the factored path");
    constexpr int STRIDE = STAGED == 2 ? GMS_SH_STRIDE_S : GMS_SH_STRIDE_V;
    __shared__ __align__(16) float s_sh[STAGED ? 4 : 1][STAGED ? GMS_SH_TILE : 4];
    __shared__ float s_f[ADAM ? 4 : 1][ADAM ? 32 * GMS_SH_FSTRIDE : 1];
    const PreArgs& a = b.f;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (!STAGED && i >= a.P) return;
    const bool inb = i < a.P;
    const bool vis = inb && b.radii[i] > 0;
    if (STAGED) {       // (only launched with shs, dshs != NULL and M == 16)
        const unsigned rows = __ballot_sync(0xffffffffu, ADAM ? inb : vis);
        if (rows) sh_tile_load<STRIDE, !ADAM>(ADAM ? b.sh_p : a.shs, blockIdx.x * blockDim.x + warp * 32, rows, lane, s_sh[warp]);
    }
    GmsPreGradOut go;
    go.dmean3D[0] = go.dmean3D[1] = go.dmean3D[2] = 0.f;
    go.dopacity = 0.f;
#pragma unroll
    for (int k = 0; k < 6; k++) go.dcov6[k] = 0.f;
    go.dscale[0] = go.dscale[1] = go.dscale[2] = 0.f;
    go.drot[0] = go.drot[1] = go.drot[2] = go.drot[3] = 0.f;
    float dm2[2] = {0.f, 0.f}, dcol[3] = {0.f, 0.f, 0.f};
    float4* dsh4 = (!STAGED && b.dshs && ((a.M * 3) & 3) == 0) ? reinterpret_cast<float4*>(b.dshs + (size_t)i * a.M * 3) : nullptr;
    float dsh[48];
    const int nfM = 3 * a.M;
    if (vis) {
        float view[16], proj[16];
#pragma unroll
        for (int k = 0; k < 16; k++) { view[k] = __ldg(a.view + k); proj[k] = __ldg(a.proj + k); }
        const float mean[3] = {a.means[3 * i], a.means[3 * i + 1], a.means[3 * i + 2]};
        float sc[3], rt[4];
        const float* scp = nullptr; const float* rtp = nullptr;
        if (!a.cov_pre) {
            sc[0] = a.scales[3 * i]; sc[1] = a.scales[3 * i + 1]; sc[2] = a.scales[3 * i + 2];
            const float4 q = reinterpret_cast<const float4*>(a.rots)[i];
            rt[0] = q.x; rt[1] = q.y; rt[2] = q.z; rt[3] = q.w;
            scp = sc; rtp = rt;
        }
        float cov6[6];
        const float2* c2 = reinterpret_cast<const float2*>(b.cov3D + 6 * (size_t)i);
        { const float2 u = c2[0], v = c2[1], w = c2[2]; cov6[0] = u.x; cov6[1] = u.y; cov6[2] = v.x; cov6[3] = v.y; cov6[4] = w.x; cov6[5] = w.y; }
        const float4 g0 = b.dgeom[3 * (size_t)i], g1 = b.dgeom[3 * (size_t)i + 1], g2 = b.dgeom[3 * (size_t)i + 2];
        GmsPreGradIn gi;
        gi.dmean2D[0] = g0.x; gi.dmean2D[1] = g0.y;
        gi.dconic[0] = g0.z; gi.dconic[1] = g0.w; gi.dconic[2] = g1.x;
        gi.dopac = g1.y;
        gi.dcolor[0] = g1.z; gi.dcolor[1] = g1.w; gi.dcolor[2] = g2.x;
        gi.dinvdepth = g2.y;
        dm2[0] = g0.x; dm2[1] = g0.y;
        dcol[0] = gi.dcolor[0]; dcol[1] = gi.dcolor[1]; dcol[2] = gi.dcolor[2];
        gms_preprocess_backward_geom(mean, scp, rtp, cov6, a.opac[i], view, proj, a.tanfovx, a.tanfovy, a.focal_x,
                                     a.focal_y, a.mod, a.antialiasing, gi, go);
        if (STAGED == 2) {
            const uint32_t clb = b.clamped[i];
            const uint8_t cl[3] = {(uint8_t)(clb & 1u), (uint8_t)((clb >> 1) & 1u), (uint8_t)((clb >> 2) & 1u)};
            const float campos[3] = {__ldg(a.campos), __ldg(a.campos + 1), __ldg(a.campos + 2)};
            float* rowp = &s_sh[warp][lane * STRIDE];
            gms_sh_backward(a.D, 16, mean, campos, rowp, gi.dcolor, cl, rowp, go.dmean3D);
        } else if (a.shs && (b.dshs || FACT)) {
            float sh[48];
            const int nf = 3 * (a.D + 1) * (a.D + 1);
            const float* row = a.shs + (size_t)i * a.M * 3;
            if (STAGED) {
#pragma unroll
                for (int k = 0; k < 12; k++) {
                    if (4 * k < nf) {
                        const float4 v = *reinterpret_cast<const float4*>(&s_sh[warp][lane * STRIDE + 4 * k]);
                        sh[4 * k] = v.x; sh[4 * k + 1] = v.y; sh[4 * k + 2] = v.z; sh[4 * k + 3] = v.w;
                    }
                }
            } else if (((a.M * 3) & 3) == 0) {
                const float4* r4 = reinterpret_cast<const float4*>(row);
#pragma unroll
                for (int k = 0; k < 12; k++) {
                    if (4 * k < nf) {
                        const float4 v = __ldg(r4 + k);
                        sh[4 * k] = v.x; sh[4 * k + 1] = v.y; sh[4 * k + 2] = v.z; sh[4 * k + 3] = v.w;
                    }
                }
            } else {
#pragma unroll
                for (int k = 0; k < 48; k++) if (k < nf) sh[k] = __ldg(row + k);
            }
            const uint32_t clb = b.clamped[i];
            const uint8_t cl[3] = {(uint8_t)(clb & 1u), (uint8_t)((clb >> 1) & 1u), (uint8_t)((clb >> 2) & 1u)};
            const float campos[3] = {__ldg(a.campos), __ldg(a.campos + 1), __ldg(a.campos + 2)};
            gms_sh_backward(a.D, a.M < 16 ? a.M : 16, mean, campos, sh, gi.dcolor, cl, FACT ? nullptr : dsh, go.dmean3D);
            if (FACT) { dcol[0] = cl[0] ? 0.f : dcol[0]; dcol[1] = cl[1] ? 0.f : dcol[1]; dcol[2] = cl[2] ? 0.f : dcol[2]; }
        }
    }
    if (FACT) {
        if (inb && (!ADAM || b.dcol_sh)) { b.dcol_sh[3 * i] = dcol[0]; b.dcol_sh[3 * i + 1] = dcol[1]; b.dcol_sh[3 * i + 2] = dcol[2]; }
    }
    if (ADAM) {
        float* f = s_f[warp] + lane * GMS_SH_FSTRIDE;
        if (inb && !(dcol[0] == 0.f && dcol[1] == 0.f && dcol[2] == 0.f)) {
            float B[16];
            sh_grad_basis(a.D, a.means[3 * i], a.means[3 * i + 1], a.means[3 * i + 2], a.campos, B);
#pragma unroll
            for (int k = 0; k < 16; k++) f[k] = B[k];
            f[16] = dcol[0]; f[17] = dcol[1]; f[18] = dcol[2];
        } else {
#pragma unroll
            for (int k = 0; k < GMS_SH_FSTRIDE; k++) f[k] = 0.f;
        }
        sh_adam_warp<ADAM_IEEE>(b.sh_adam, b.sh_p, b.sh_m, b.sh_v, a.P, blockIdx.x * blockDim.x + warp * 32, lane, s_sh[warp], s_f[warp]);
    }
    if (STAGED && FACT) { if (!inb) return; }
    else if (STAGED) {       // gradient rows -> the warp's tile (zeros for culled Gaussians) -> coalesced 128-bit stores
        if (STAGED == 2) {
            if (!vis) {
#pragma unroll
                for (int k = 0; k < 48; k++) s_sh[warp][lane * STRIDE + k] = 0.f;
            }
        } else {
#pragma unroll
            for (int k = 0; k < 12; k++) {      // gms_sh_backward fills all 16 coefficients (zeros above the active degree)
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (vis) v = make_float4(dsh[4 * k], dsh[4 * k + 1], dsh[4 * k + 2], dsh[4 * k + 3]);
                *reinterpret_cast<float4*>(&s_sh[warp][lane * STRIDE + 4 * k]) = v;
            }
        }
        sh_tile_store<STRIDE>(b.dshs, blockIdx.x * blockDim.x + warp * 32, a.P, lane, s_sh[warp]);
        if (!inb) return;
    }
    // every output row is written (zeros for culled Gaussians): callers hand in torch.empty buffers
    b.dmeans3D[3 * i] = go.dmean3D[0]; b.dmeans3D[3 * i + 1] = go.dmean3D[1]; b.dmeans3D[3 * i + 2] = go.dmean3D[2];
    b.dmeans2D[3 * i] = dm2[0]; b.dmeans2D[3 * i + 1] = dm2[1]; b.dmeans2D[3 * i + 2] = 0.f;
    if (b.dopac_raw) { const float y = vis ? a.opac[i] : 0.f; b.dopac_raw[i] = go.dopacity * y * (1.0f - y); }
    else b.dopac[i] = go.dopacity;
    if (!STAGED && b.dshs) {
        if (dsh4) {
#pragma unroll
            for (int k = 0; k < 12; k++)
                if (4 * k < nfM) {
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (vis) v = make_float4(dsh[4 * k], dsh[4 * k + 1], dsh[4 * k + 2], dsh[4 * k + 3]);
                    dsh4[k] = v;
                }
        } else {
            float* row = b.dshs + (size_t)i * a.M * 3;
            for (int k = 0; k < nfM; k++) row[k] = (vis && k < 48) ? dsh[k] : 0.f;
        }
    }
    if (b.dcolors_pre) { b.dcolors_pre[3 * i] = dcol[0]; b.dcolors_pre[3 * i + 1] = dcol[1]; b.dcolors_pre[3 * i + 2] = dcol[2]; }
    if (b.dscales) { b.dscales[3 * i] = go.dscale[0]; b.dscales[3 * i + 1] = go.dscale[1]; b.dscales[3 * i + 2] = go.dscale[2]; }
    if (b.drots) reinterpret_cast<float4*>(b.drots)[i] = make_float4(go.drot[0], go.drot[1], go.drot[2], go.drot[3]);
    if (b.dcov_pre) {
#pragma unroll
        for (int k = 0; k < 6; k++) b.dcov_pre[6 * (size_t)i + k] = go.dcov6[k];
    }
}

__global__ void k_set_u32(uint32_t* p, uint32_t v) { *p = v; }

__global__ void k_mark_visible(int P, const float* __restrict__ means, const float* __restrict__ view, uint8_t* __restrict__ present) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float v[16];
#pragma unroll
    for (int k = 0; k < 16; k++) v[k] = __ldg(view + k);
    float pv[3];
    gms_xform4x3(v, means[3 * i], means[3 * i + 1], means[3 * i + 2], pv);
    present[i] = pv[2] > GMS_NEAR ? 1 : 0;
}

// debug: unpack the packed records into the stock layouts
__global__ void k_unpack(int P, const float4* __restrict__ rec, const uint32_t* __restrict__ clamped, const uint32_t* __restrict__ dkey,
                         const int* radii, float* means2D, float* depths, float* conic_opacity, float* rgb, uint8_t* cl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const bool vis = radii[i] > 0;
    float4 a = make_float4(0, 0, 0, 0), b = a, c = a; uint32_t m = 0;
    if (vis) { a = rec[3 * (size_t)i]; b = rec[3 * (size_t)i + 1]; c = rec[3 * (size_t)i + 2]; m = clamped[i]; }
    if (means2D) { means2D[2 * i] = a.x; means2D[2 * i + 1] = a.y; }
    if (depths) depths[i] = vis ? __uint_as_float(dkey[i]) : 0.f;   // the exact bits used as the sort key
    if (conic_opacity) { conic_opacity[4 * i] = a.z; conic_opacity[4 * i + 1] = a.w; conic_opacity[4 * i + 2] = b.x; conic_opacity[4 * i + 3] = b.y; }
    if (rgb) { rgb[3 * i] = b.z; rgb[3 * i + 1] = b.w; rgb[3 * i + 2] = c.x; }
    if (cl) { cl[3 * i] = m & 1u; cl[3 * i + 1] = (m >> 1) & 1u; cl[3 * i + 2] = (m >> 2) & 1u; }
}

struct TilesInOrder {   // tiles_touched permuted into depth order, evaluated on the fly by the scan
    const uint32_t* tiles; const uint32_t* order;
    __host__ __device__ __forceinline__ uint32_t operator()(const uint32_t& j) const { return tiles[order[j]]; }
};
