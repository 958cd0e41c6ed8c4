// gms_kernels.cu -- kernels + C ABI of libgms_b200.so (see include/gms_b200.h for what each entry point replaces).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 --shared -Xcompiler -fPIC
// No torch headers; PyTorch only provides memory and the stream on the Python side.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "../../include/gms_b200.h"
#define GMS_BRANCHFREE_DIV 1        // the product: branch-free correctly-rounded division / sqrt where operands are provably normal (gms_common.cuh)
#include "gms_common.cuh"
#include "gms_preprocess.cuh"
#include "gms_expand.cuh"
#include "gms_composite_fwd.cuh"
#include "gms_composite_bwd.cuh"
#include "gms_loss.cuh"
#include "gms_sort.cuh"
#include "gms_binning.cuh"
#include "gms_image.cuh"
#include "gms_free.cuh"
#include "gms_knn.cuh"

// ------------------------------------------------------------------------------------------ host state
static thread_local char g_err[512] = "";
static int64_t g_launches = 0;
// Defaults chosen on an H100 SXM (400 W) at 1M mesh-Gaussians / 1080p: step time with each alternative, default = 2.61-2.66 ms
// over five interleaved runs, measured with the earlier float2-pair composite backward; 2.45 ms with the scalar one (DESIGN.md 3.7).
static int g_opt_warp_emit = 1;    // (emit + sort path) warp-cooperative duplicate emission for large rects (0: 2.65 ms)
static int g_opt_fwd = 2;          // composite forward: 2 scalar (default; writes the survivor lists), 3 float2 pairs (bit-identical; 2.81 ms)
static int g_opt_bwd = 5;          // composite backward: 5 survivor-list driven (default), 3 predecessor (streams the whole tile list; 2.73 ms)
static int g_opt_adam_sh_ieee = 0;  // k_adam_sh: 1 = nvcc's sqrtf / division with slow-path branches (A/B arm of the branch-free sequences)
static int g_opt_key16 = 1;        // tile sort on 16-bit keys when T <= 65535 (0: always 32-bit keys; 2.66 ms)
static int g_opt_bwd_minb = 6;     // __launch_bounds__ min CTAs/SM of the backward kernels (6: 75 regs, 2.445-2.458 ms; 4: 76, 2.449;
                                   // 8: 64, 2.449; 5: 76)
static int g_opt_tile_order = 1;   // launch tiles longest list first (0: 2.79 ms)
static int g_opt_sh_staged = 1;     // preprocess fwd/bwd: SH rows through a per-warp shared-memory tile (coalesced 128-bit accesses);
                                    // 0: direct (2.66 ms), 1: tile + register rows, 2: bwd in place in the tile (2.63 ms)
static int g_opt_pre_bwd_minb = 4;  // k_preprocess_bwd min CTAs/SM (1: 2.67 ms, 3: 2.67 ms, 4: default)
static int g_opt_expand_staged = 1; // expansion kernels, per-Gaussian streams staged through shared memory (coalesced): bit 0 forward
                                    // (0: 2.74 ms), bit 1 backward (3: 2.67 ms, off)
static int g_opt_expand_wide = 1;  // expansion kernels, one warp per face (k_expand_wide_*): 0 never, 1 softmax weights with K >=
                                    // GMS_EXP_WIDE_MIN_K (default; relu meshes keep the per-thread kernels), 2 always (A/B runs, tests)
static int g_opt_sort = 0;         // depth sort (and the emit + sort path's tile sort): 0 cub::DeviceRadixSort, 1 hand-written radix sort
                                   //    with device-side N clamped to the capacity (gms_sort.cuh; bit-identical order through the
                                   //    synchronising entry points and the sync-free frame; 2.67-2.70 ms against 2.40-2.42 ms
                                   //    for the default with the current build, DESIGN.md 3.7)
static int g_opt_bin = 0;          // tile binning: 0 emit in depth order + ONE stable radix sort on the tile bits (default),
                                   //               1 cooperative counting kernel without any sort over the duplicates (gms_binning.cuh;
                                   //                 2.92 ms -- kept selectable, parity-tested)
static uint32_t* g_pinned = nullptr;
static int g_sm_count = 0;
static int g_bin_smem_optin = 0;
static int sm_count() {
    if (!g_sm_count) {
        int dev = 0; cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&g_bin_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (g_sm_count <= 0) g_sm_count = 132;   // H100 SXM
    }
    return g_sm_count;
}

// Optional per-kernel timing with CUDA events recorded on the launching stream (bench.py's roofline numbers).
enum { K_PRE_FWD = 0, K_SORT_P, K_SCAN, K_EMIT, K_SORT_N, K_RANGES, K_COMP_FWD, K_COMP_BWD, K_PRE_BWD, K_EXP_FWD, K_EXP_BWD, K_LOSS_STATS, K_LOSS_GRAD, K_ADAM, K_MISC,
       K_METRICS, K_METRICS_FIN, K_COUNT };
static const char* const g_kernel_names[K_COUNT] = {"preprocess_fwd", "cub_sort_depth", "cub_scan_tiles", "emit_dups", "cub_sort_tiles",
                                                    "tile_ranges", "composite_fwd", "composite_bwd", "preprocess_bwd", "expand_fwd",
                                                    "expand_bwd", "ssim_stats", "ssim_grad", "adam", "misc",
                                                    "image_metrics", "metrics_finalize"};
static int g_opt_time = 0;
struct TimedSpan { int id; cudaEvent_t a, b; };
static TimedSpan g_spans[1 << 15];
static int g_nspans = 0;
static double g_ktime_ms[K_COUNT];
static int64_t g_kcount[K_COUNT];

static void span_begin(int id, cudaStream_t st) {
    if (!g_opt_time || g_nspans >= (1 << 15)) return;
    TimedSpan& s = g_spans[g_nspans];
    s.id = id;
    cudaEventCreate(&s.a); cudaEventCreate(&s.b);
    cudaEventRecord(s.a, st);
}
static void span_end(cudaStream_t st) {
    if (!g_opt_time || g_nspans >= (1 << 15)) return;
    cudaEventRecord(g_spans[g_nspans].b, st);
    g_nspans++;
}
static void spans_collect() {
    for (int i = 0; i < g_nspans; i++) {
        float ms = 0.f;
        cudaEventSynchronize(g_spans[i].b);
        if (cudaEventElapsedTime(&ms, g_spans[i].a, g_spans[i].b) == cudaSuccess) { g_ktime_ms[g_spans[i].id] += ms; g_kcount[g_spans[i].id]++; }
        cudaEventDestroy(g_spans[i].a); cudaEventDestroy(g_spans[i].b);
    }
    g_nspans = 0;
}

static int set_err(int code, const char* fmt, const char* a = "", const char* b = "") {
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}

#define GMS_CUDA(call)                                                                         \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess) return set_err(GMS_E_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); \
    } while (0)

#define GMS_AFTER_LAUNCH(name, debug, stream)                                                  \
    do {                                                                                       \
        g_launches++;                                                                          \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ == cudaSuccess && (debug)) e__ = cudaStreamSynchronize(stream);                \
        if (e__ != cudaSuccess) return set_err(GMS_E_CUDA, "kernel %s: %s", name, cudaGetErrorString(e__)); \
    } while (0)

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

static inline void* aligned_base_c(void* p) { return reinterpret_cast<void*>(align_up(reinterpret_cast<size_t>(p))); }

template <typename T>
static T* carve(char*& p, size_t count) {
    T* r = reinterpret_cast<T*>(p);
    p += align_up(count * sizeof(T));
    return r;
}

struct GeomLayout {
    float4* rec;        // [3P] packed splat records
    float* cov3D;       // [6P]
    uint32_t* clamped;  // [P] bits 0..2
    uint32_t* tiles;    // [P]
    uint32_t* dkey;     // [P] depth bits (0xFFFFFFFF when culled)
    uint32_t* idx;      // [P] iota
    uint32_t* dkey_s;   // [P]
    uint32_t* order;    // [P] Gaussian ids sorted by (depth bits, id)   (cub path; own sort: ping-pong pair 0)
    uint32_t* dkey_t;   // [P] ping-pong pair 1 of the hand-written sort
    uint32_t* order_t;  // [P]
    void* sort_temp;    // histograms of the hand-written sort
    uint32_t* offs;     // [P] inclusive scan of tiles in `order`
    float4* dgeom;      // [3P] backward accumulators
    uint32_t* counters; // [64]: 0 N, 1 overflow flag (k_bin_tiles), 2 visible Gaussians, 3 sum of tiles_touched (k_preprocess_fwd)
    uint2* rect;        // [P] packed tile rectangles (x0 | y0 << 16, x1 | y1 << 16), empty when culled
    void* cub_temp;
    size_t cub_bytes;
    size_t total;
};

struct TilesInOrder {   // tiles_touched permuted into depth order, evaluated on the fly by the scan
    const uint32_t* tiles; const uint32_t* order;
    __host__ __device__ __forceinline__ uint32_t operator()(const uint32_t& j) const { return tiles[order[j]]; }
};

static size_t cub_temp_geom(int P) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, P, 0, 32);
    auto it = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), TilesInOrder{nullptr, nullptr});
    cub::DeviceScan::InclusiveSum(nullptr, b, it, (uint32_t*)nullptr, P);
    return a > b ? a : b;
}

static GeomLayout geom_layout(void* base, int P) {
    GeomLayout L;
    char* p = reinterpret_cast<char*>(base);
    const size_t Pn = (size_t)(P > 0 ? P : 1);
    L.rec = carve<float4>(p, 3 * Pn);
    L.cov3D = carve<float>(p, 6 * Pn);
    L.clamped = carve<uint32_t>(p, Pn);
    L.tiles = carve<uint32_t>(p, Pn);
    L.dkey = carve<uint32_t>(p, Pn);
    L.idx = carve<uint32_t>(p, Pn);
    L.dkey_s = carve<uint32_t>(p, Pn);
    L.order = carve<uint32_t>(p, Pn);
    L.offs = carve<uint32_t>(p, Pn);
    L.dkey_t = carve<uint32_t>(p, Pn);
    L.order_t = carve<uint32_t>(p, Pn);
    L.sort_temp = p;
    p += align_up(gms_sort_temp_bytes((int64_t)Pn));
    L.dgeom = carve<float4>(p, 3 * Pn);
    L.counters = carve<uint32_t>(p, 64);
    L.rect = carve<uint2>(p, Pn);
    L.cub_bytes = cub_temp_geom((int)Pn);
    L.cub_temp = p;
    p += align_up(L.cub_bytes);
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

struct ImageLayout {
    float* final_T; int* n_contrib; int* tile_last; int2* ranges; int* tile_order; uint32_t* binM; uint32_t* bin_total; uint32_t* nsurv; size_t total;
};

static ImageLayout image_layout(void* base, int W, int H) {
    ImageLayout L;
    char* p = reinterpret_cast<char*>(base);
    const size_t HW = (size_t)W * H;
    const size_t T = (size_t)((W + GMS_TILE - 1) / GMS_TILE) * ((H + GMS_TILE - 1) / GMS_TILE);
    L.final_T = carve<float>(p, HW);
    L.n_contrib = carve<int>(p, HW);
    L.tile_last = carve<int>(p, T);
    L.ranges = carve<int2>(p, T);
    L.tile_order = carve<int>(p, T);
    L.binM = carve<uint32_t>(p, T * (size_t)(2 * sm_count()));  // k_bin_tiles: per-CTA tile counts (up to 2 CTAs per SM)
    L.bin_total = carve<uint32_t>(p, T);
    L.nsurv = carve<uint32_t>(p, 4 * T);                      // survivors per (tile, quad), written by k_composite_fwd2<true>
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

struct BinLayout {
    uint32_t* keys_in; uint32_t* vals_in; uint32_t* keys_out; uint32_t* vals_out; void* cub_temp; size_t cub_bytes; void* sort_temp;
    uint32_t* surv;     // [4N] per-quad survivor lists (present when the forward emits them; counted in total_with_lists only)
    size_t total, total_with_lists;
};

static BinLayout bin_layout(void* base, int64_t N) {
    BinLayout L;
    char* p = reinterpret_cast<char*>(base);
    const size_t Nn = (size_t)(N > 0 ? N : 1);
    L.keys_in = carve<uint32_t>(p, Nn);
    L.vals_in = carve<uint32_t>(p, Nn);
    L.keys_out = carve<uint32_t>(p, Nn);
    L.vals_out = carve<uint32_t>(p, Nn);
    // cub's temporary storage grows with the number of digit passes: the 32-bit-key sort is sized for all 32 key bits, since
    // grids above 65535 tiles sort on 17 or more (sized for 16, the sort rejected its storage at 4096x4096)
    size_t a = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)Nn, 0, 32);
    size_t a16 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a16, (uint16_t*)nullptr, (uint16_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)Nn, 0, 16);
    a = a16 > a ? a16 : a;
    L.cub_bytes = a;
    L.cub_temp = p;
    p += align_up(a);
    L.sort_temp = p;
    p += align_up(gms_sort_temp_bytes((int64_t)Nn));
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    L.surv = carve<uint32_t>(p, 4 * Nn);
    L.total_with_lists = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

__global__ void k_set_u32(uint32_t* p, uint32_t v) { *p = v; }

// ------------------------------------------------------------------------------------------ kernels
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

// ------------------------------------------------------------------------------------------ expansion kernels
// One thread per face.  The per-Gaussian streams (K rows per face: 36-48 B per thread, i.e. a 36-48 B stride between
// lanes) are staged through shared memory: the block copies its contiguous slice of every stream with fully coalesced
// accesses, the per-face maths then reads / writes shared memory (gms_expand_face_* with fl = slot in the block).
// STAGED = false is the direct variant (option "expand_staged" = 0, and whenever K makes the staging exceed 48 KB).
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

// floats of shared memory per Gaussian row (host side: sizing the launch)
static int exp_fwd_stage_width(const gms_expand_args& a) {
    return 3 + 1 + (a.alpha ? 3 : 0) + (a.xyz ? 3 : 0) + (a.scaling_log ? 3 : 0) + (a.scaling_act ? 3 : 0) +
           (a.rotation_raw ? 4 : 0) + (a.rotation_act ? 4 : 0);
}
static int exp_bwd_stage_width(const gms_expand_grads& g) {
    return 3 + 1 + (g.dL_dxyz ? 3 : 0) + (g.dL_dscaling_log ? 3 : 0) + (g.dL_dscaling_act ? 3 : 0) +
           (g.dL_drotation_raw ? 4 : 0) + (g.dL_drotation_act ? 4 : 0) + (g.dL_dalpha_raw ? 3 : 0) + (g.dL_dscale_raw ? 1 : 0);
}

template <int ACT>
__device__ __forceinline__ void expand_face_fwd(const gms_expand_args& a, int f, int fl) {
    if constexpr (ACT == GMS_ALPHA_RELU) gms_expand_face_fwd_relu(a, f, fl);
    else gms_expand_face_fwd_act<ACT>(a, f, fl);
}
template <int ACT>
__device__ __forceinline__ void expand_face_bwd(const gms_expand_args& a, const gms_expand_grads& g, int f, int fl) {
    if constexpr (ACT == GMS_ALPHA_RELU) gms_expand_face_bwd_relu(a, g, f, fl);
    else gms_expand_face_bwd_act<ACT>(a, g, f, fl);
}

template <bool STAGED, int ACT>
__device__ __forceinline__ void expand_fwd_block(const gms_expand_args& a) {
    const int f0 = blockIdx.x * GMS_EXP_BLOCK, f = f0 + threadIdx.x;
    if (!STAGED) {
        if (f < a.F) expand_face_fwd<ACT>(a, f, f);
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
    if (f < a.F) expand_face_fwd<ACT>(l, f, threadIdx.x);
    __syncthreads();
    exp_stage_flush(a.alpha, l.alpha, 3, g0, ng);
    exp_stage_flush(a.xyz, l.xyz, 3, g0, ng);
    exp_stage_flush(a.scaling_log, l.scaling_log, 3, g0, ng);
    exp_stage_flush(a.scaling_act, l.scaling_act, 3, g0, ng);
    exp_stage_flush(a.rotation_raw, l.rotation_raw, 4, g0, ng);
    exp_stage_flush(a.rotation_act, l.rotation_act, 4, g0, ng);
}

template <bool STAGED>
__global__ void __launch_bounds__(GMS_EXP_BLOCK) k_expand_fwd(gms_expand_args a) { expand_fwd_block<STAGED, GMS_ALPHA_RELU>(a); }
template <bool STAGED>
__global__ void __launch_bounds__(GMS_EXP_BLOCK) k_expand_softmax_fwd(gms_expand_args a) { expand_fwd_block<STAGED, GMS_ALPHA_SOFTMAX>(a); }

template <bool STAGED, int ACT>
__device__ __forceinline__ void expand_bwd_block(const gms_expand_args& a, const gms_expand_grads& g) {
    const int f0 = blockIdx.x * GMS_EXP_BLOCK, f = f0 + threadIdx.x;
    if (!STAGED) {
        if (f < a.F) expand_face_bwd<ACT>(a, g, f, f);
        return;
    }
    extern __shared__ float4 exp_smem4[];
    float* sm = reinterpret_cast<float*>(exp_smem4);
    const int nf = min(GMS_EXP_BLOCK, a.F - f0), ng = nf * a.K, cap = GMS_EXP_BLOCK * a.K;
    const size_t g0 = (size_t)f0 * a.K;
    gms_expand_args l = a;
    gms_expand_grads lg = g;
    l.alpha_raw = exp_stage_in(a.alpha_raw, 3, g0, ng, cap, sm);
    l.scale_raw = exp_stage_in(a.scale_raw, 1, g0, ng, cap, sm);
    lg.dL_dxyz = exp_stage_in(g.dL_dxyz, 3, g0, ng, cap, sm);
    lg.dL_dscaling_log = exp_stage_in(g.dL_dscaling_log, 3, g0, ng, cap, sm);
    lg.dL_dscaling_act = exp_stage_in(g.dL_dscaling_act, 3, g0, ng, cap, sm);
    lg.dL_drotation_raw = exp_stage_in(g.dL_drotation_raw, 4, g0, ng, cap, sm);
    lg.dL_drotation_act = exp_stage_in(g.dL_drotation_act, 4, g0, ng, cap, sm);
    lg.dL_dalpha_raw = exp_stage_out(g.dL_dalpha_raw, 3, cap, sm);
    lg.dL_dscale_raw = exp_stage_out(g.dL_dscale_raw, 1, cap, sm);
    __syncthreads();
    if (f < a.F) expand_face_bwd<ACT>(l, lg, f, threadIdx.x);     // per-face outputs (dL_dtriangles, vertex atomics) stay global
    __syncthreads();
    exp_stage_flush(g.dL_dalpha_raw, lg.dL_dalpha_raw, 3, g0, ng);
    exp_stage_flush(g.dL_dscale_raw, lg.dL_dscale_raw, 1, g0, ng);
}

template <bool STAGED>
__global__ void __launch_bounds__(GMS_EXP_BLOCK) k_expand_bwd(gms_expand_args a, gms_expand_grads g) {
    expand_bwd_block<STAGED, GMS_ALPHA_RELU>(a, g);
}
template <bool STAGED>
__global__ void __launch_bounds__(GMS_EXP_BLOCK) k_expand_softmax_bwd(gms_expand_args a, gms_expand_grads g) {
    expand_bwd_block<STAGED, GMS_ALPHA_SOFTMAX>(a, g);
}

// Splat-parallel expansion for many splats per face (gs_flame: K = 100 on ~10k faces).  One warp per face: every lane reads
// the face and evaluates its frame and quaternion in lockstep (one instruction stream per face, as cheap as one lane
// computing them and broadcasting the result, without the shuffles), then lane j handles splats j, j + 32, ...: consecutive
// lanes touch consecutive rows, so every per-Gaussian stream is read and written coalesced without staging.  Each splat is
// the per-thread kernel's gms_expand_splat_* call, so the forward is bit-identical to it.  The backward sums each lane's
// dt / dq / ds1 / ds2 partials over its splats, reduces them across the warp (butterfly), and lane 0 finishes the face: one
// set of vertex atomics per face, as in the per-thread kernel.  Only the order of the sum over K differs.
constexpr int GMS_EXP_WIDE_BLOCK = 128;                     // 4 faces per block
constexpr int GMS_EXP_WIDE_MIN_K = 16;                      // expand_wide = 1: softmax weights with K >= this (DESIGN.md 4.5)

template <int ACT>
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
    for (int k = lane; k < a.K; k += 32) gms_expand_splat_fwd<ACT>(a, s, (size_t)f * a.K + k);
}

template <int ACT>
__global__ void __launch_bounds__(GMS_EXP_WIDE_BLOCK) k_expand_wide_bwd(gms_expand_args a, gms_expand_grads g) {
    const int f = blockIdx.x * (GMS_EXP_WIDE_BLOCK / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= a.F) return;                                   // whole warps: f is uniform across the warp
    GmsFaceState s;
    gms_expand_face_load(a, f, s);
    gms_expand_face_frame(a, s);
    float acc[15];                                          // dt[9], dq[4], ds1, ds2
#pragma unroll
    for (int i = 0; i < 15; i++) acc[i] = 0.f;
    for (int k = lane; k < a.K; k += 32) gms_expand_splat_bwd<ACT>(a, g, s, (size_t)f * a.K + k, acc, acc + 9, acc[13], acc[14]);
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

extern "C" int gms_loss_scratch_bytes(int32_t C, int32_t H, int32_t W, size_t* bytes);

// ------------------------------------------------------------------------------------------ whole-frame orchestration

struct FrameLayout {
    float* xyz; float* scales; float* rots; float* opac; int32_t* radii; float* image; float* invdepth; float* dimage;
    float* d_xyz; float* d_m2d; float* d_opac; float* d_scales; float* d_rots; float* loss_scratch; size_t loss_bytes; size_t total;
};

static FrameLayout frame_layout(void* base, int P, int W, int H) {
    FrameLayout L;
    char* p = reinterpret_cast<char*>(base);
    const size_t Pn = (size_t)(P > 0 ? P : 1), HW = (size_t)W * H;
    L.xyz = carve<float>(p, 3 * Pn); L.scales = carve<float>(p, 3 * Pn); L.rots = carve<float>(p, 4 * Pn); L.opac = carve<float>(p, Pn);
    L.radii = carve<int32_t>(p, Pn);
    L.image = carve<float>(p, 3 * HW); L.invdepth = carve<float>(p, HW); L.dimage = carve<float>(p, 3 * HW);
    L.d_xyz = carve<float>(p, 3 * Pn); L.d_m2d = carve<float>(p, 3 * Pn); L.d_opac = carve<float>(p, Pn);
    L.d_scales = carve<float>(p, 3 * Pn); L.d_rots = carve<float>(p, 4 * Pn);
    size_t lb = 0;
    gms_loss_scratch_bytes(3, H, W, &lb);
    L.loss_scratch = reinterpret_cast<float*>(p); L.loss_bytes = lb;
    p += align_up(lb);
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

// ------------------------------------------------------------------------------------------ C ABI
extern "C" {

int gms_loss_scratch_bytes(int32_t C, int32_t H, int32_t W, size_t* bytes) {
    if (C <= 0 || H <= 0 || W <= 0 || !bytes) return set_err(GMS_E_ARG, "gms_loss_scratch_bytes: bad sizes%s%s");
    *bytes = align_up(sizeof(float) * 3 * (size_t)C * H * W) + 256 + 256;
    return GMS_OK;
}

static GmsGaussWin ssim_window() {
    GmsGaussWin win;    // utils/loss_utils.py:23-25: exp(-(x-5)^2 / (2*1.5^2)) in fp32, normalised
    float sum = 0.f;
    for (int k = 0; k < 11; k++) { win.g[k] = (float)exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)); sum += win.g[k]; }
    for (int k = 0; k < 11; k++) win.g[k] /= sum;
    return win;
}

int gms_l1_ssim_loss(const gms_loss_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->img || !a->gt || !a->loss || !a->scratch) return set_err(GMS_E_ARG, "gms_l1_ssim_loss: null argument%s%s");
    const int C = a->C, H = a->H, W = a->W;
    size_t need = 0;
    gms_loss_scratch_bytes(C, H, W, &need);
    if (a->scratch_bytes < need) return set_err(GMS_E_ARG, "gms_l1_ssim_loss: scratch too small%s%s");
    char* base = reinterpret_cast<char*>(aligned_base_c(a->scratch));
    float* acc = reinterpret_cast<float*>(base);
    float* dmap = reinterpret_cast<float*>(base + 256);
    const GmsGaussWin win = ssim_window();
    GMS_CUDA(cudaMemsetAsync(acc, 0, 2 * sizeof(float), st));
    dim3 grid((W + GMS_SSIM_T - 1) / GMS_SSIM_T, (H + GMS_SSIM_T - 1) / GMS_SSIM_T, C);
    span_begin(K_LOSS_STATS, st);
    k_ssim_stats<<<grid, 256, 0, st>>>(C, H, W, a->img, a->gt, win, a->dL_dimg ? dmap : nullptr, acc);
    GMS_AFTER_LAUNCH("ssim_stats", 0, st);
    span_end(st);
    const float inv_n = 1.0f / ((float)C * (float)H * (float)W);
    k_loss_finalize<<<1, 1, 0, st>>>(acc, inv_n, a->lambda_dssim, a->loss);
    GMS_AFTER_LAUNCH("loss_finalize", 0, st);
    if (a->dL_dimg) {
        span_begin(K_LOSS_GRAD, st);
        k_ssim_grad<<<grid, 256, 0, st>>>(C, H, W, a->img, a->gt, win, dmap, -a->lambda_dssim * inv_n,
                                         (1.f - a->lambda_dssim) * inv_n, a->dL_dloss, a->dL_dimg);
        GMS_AFTER_LAUNCH("ssim_grad", 0, st);
        span_end(st);
    }
    return GMS_OK;
}

static int metric_tiles(int32_t H, int32_t W) { return ((W + GMS_SSIM_T - 1) / GMS_SSIM_T) * ((H + GMS_SSIM_T - 1) / GMS_SSIM_T); }

int gms_metrics_scratch_bytes(int32_t C, int32_t H, int32_t W, size_t* bytes) {
    if (C <= 0 || C > GMS_METRIC_MAXC || H <= 0 || W <= 0 || !bytes) return set_err(GMS_E_ARG, "gms_metrics_scratch_bytes: bad sizes%s%s");
    *bytes = align_up(sizeof(float) * 3 * (size_t)C * metric_tiles(H, W)) + 256;
    return GMS_OK;
}

int gms_image_metrics(const gms_metrics_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->img || !a->gt || !a->out || !a->scratch) return set_err(GMS_E_ARG, "gms_image_metrics: null argument%s%s");
    if (a->quantize != 0 && a->quantize != 1) return set_err(GMS_E_ARG, "gms_image_metrics: quantize must be 0 or 1%s%s");
    const int C = a->C, H = a->H, W = a->W;
    size_t need = 0;
    int rc = gms_metrics_scratch_bytes(C, H, W, &need);
    if (rc) return rc;
    if (a->scratch_bytes < need) return set_err(GMS_E_ARG, "gms_image_metrics: scratch too small%s%s");
    float* part = reinterpret_cast<float*>(aligned_base_c(a->scratch));
    const GmsGaussWin win = ssim_window();
    dim3 grid((W + GMS_SSIM_T - 1) / GMS_SSIM_T, (H + GMS_SSIM_T - 1) / GMS_SSIM_T, C);
    span_begin(K_METRICS, st);
    if (a->quantize) k_image_metrics<1><<<grid, 256, 0, st>>>(C, H, W, a->img, a->gt, win, part);
    else k_image_metrics<0><<<grid, 256, 0, st>>>(C, H, W, a->img, a->gt, win, part);
    GMS_AFTER_LAUNCH("image_metrics", 0, st);
    span_end(st);
    span_begin(K_METRICS_FIN, st);
    k_metrics_finalize<<<1, 256, 0, st>>>(C, metric_tiles(H, W), 1.0 / ((double)H * (double)W), part, a->out);
    GMS_AFTER_LAUNCH("metrics_finalize", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_adam_step(const gms_adam_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->p || !a->g || !a->m || !a->v || a->n < 0 || a->nseg < 1 || a->nseg > 8 || a->step < 1)
        return set_err(GMS_E_ARG, "gms_adam_step: bad arguments%s%s");
    if (a->n == 0) return GMS_OK;
    AdamArgs k;
    k.n = a->n; k.offset = a->offset; k.p = a->p; k.g = a->g; k.m = a->m; k.v = a->v; k.nseg = a->nseg;
    const double bc1 = 1.0 - pow(a->beta1, (double)a->step);
    for (int i = 0; i < a->nseg; i++) {
        k.seg[i].end = a->seg_end[i];
        k.seg[i].lr0 = (float)((double)a->lr0[i] / bc1); k.seg[i].lr1 = (float)((double)a->lr1[i] / bc1);
        k.seg[i].inner = a->inner[i] > 0 ? a->inner[i] : 1; k.seg[i].period = a->period[i];
    }
    k.beta1 = (float)a->beta1; k.beta2 = (float)a->beta2; k.eps = (float)a->eps;
    k.omb1 = (float)(1.0 - a->beta1); k.omb2 = (float)(1.0 - a->beta2);
    k.bc2_sqrt = (float)sqrt(1.0 - pow(a->beta2, (double)a->step));
    k.zero_grad = a->zero_grad; k.zero_end = a->zero_end;
    const long long nthreads = (a->n + 3) / 4;
    span_begin(K_ADAM, st);
    k_adam<<<(unsigned)((nthreads + 255) / 256), 256, 0, st>>>(k);
    GMS_AFTER_LAUNCH("adam", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_image_quantize(const float* chw, uint8_t* out, int32_t C, int32_t H, int32_t W, int32_t row_prefix, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!chw || !out || C <= 0 || C > 4 || H <= 0 || W <= 0 || row_prefix < 0 || row_prefix > 16) return set_err(GMS_E_ARG, "gms_image_quantize: bad arguments%s%s");
    k_image_quantize<<<dim3((W + 255) / 256, H), 256, 0, st>>>(chw, out, C, H, W, row_prefix);
    GMS_AFTER_LAUNCH("image_quantize", 0, st);
    return GMS_OK;
}

int gms_image_dequantize(const uint8_t* src, int32_t src_is_hwc, float* chw, int32_t C, int32_t H, int32_t W, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!src || !chw || C <= 0 || C > 4 || H <= 0 || W <= 0) return set_err(GMS_E_ARG, "gms_image_dequantize: bad arguments%s%s");
    k_image_dequantize<<<dim3((W + 255) / 256, H), 256, 0, st>>>(src, src_is_hwc, chw, C, H, W);
    GMS_AFTER_LAUNCH("image_dequantize", 0, st);
    return GMS_OK;
}

int gms_image_composite_rgba(const uint8_t* rgba, uint8_t* rgb, int32_t H, int32_t W, int32_t white_background, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!rgba || !rgb || H <= 0 || W <= 0 || (white_background != 0 && white_background != 1) ||
        reinterpret_cast<size_t>(rgba) % 4 != 0)
        return set_err(GMS_E_ARG, "gms_image_composite_rgba: bad arguments%s%s");
    const long long npix = (long long)H * W;
    k_image_composite_rgba<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uchar4*>(rgba), rgb, npix,
                                                                           white_background ? 1.0 : 0.0);
    GMS_AFTER_LAUNCH("image_composite_rgba", 0, st);
    return GMS_OK;
}

int gms_image_resize_u8(const gms_resize_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->src || !a->dst || a->C != 3 || a->in_w <= 0 || a->in_h <= 0 || a->out_w <= 0 || a->out_h <= 0 ||
        a->out_w > 65535 * 256 || a->out_h > 65535 || a->in_h > 65535)
        return set_err(GMS_E_ARG, "gms_image_resize_u8: bad sizes%s%s");
    const bool horiz = a->out_w != a->in_w, vert = a->out_h != a->in_h;
    if ((horiz && (!a->bounds_h || !a->coeffs_h || a->ksize_h <= 0)) || (vert && (!a->bounds_v || !a->coeffs_v || a->ksize_v <= 0)))
        return set_err(GMS_E_ARG, "gms_image_resize_u8: missing coefficient table%s%s");
    if (!horiz && !vert) {      // Image.resize to the same size is a copy
        GMS_CUDA(cudaMemcpyAsync(a->dst, a->src, (size_t)a->in_w * a->in_h * 3, cudaMemcpyDeviceToDevice, st));
        return GMS_OK;
    }
    if (horiz && vert) {        // the horizontal pass covers only the source rows the vertical pass reads
        if (a->row0 < 0 || a->rows <= 0 || a->row0 + a->rows > a->in_h || !a->scratch ||
            a->scratch_bytes < (size_t)a->out_w * a->rows * 3)
            return set_err(GMS_E_ARG, "gms_image_resize_u8: bad row range or scratch too small%s%s");
    }
    if (horiz) {
        uint8_t* out = vert ? a->scratch : a->dst;
        const int row0 = vert ? a->row0 : 0, rows = vert ? a->rows : a->in_h;
        k_resize_h_u8<<<dim3((a->out_w + 255) / 256, rows), 256, 0, st>>>(a->src, a->in_w, out, a->out_w, row0, a->bounds_h,
                                                                          a->coeffs_h, a->ksize_h);
        GMS_AFTER_LAUNCH("resize_h_u8", 0, st);
    }
    if (vert) {
        const uint8_t* in = horiz ? a->scratch : a->src;
        const int row0 = horiz ? a->row0 : 0;
        k_resize_v_u8<<<dim3((a->out_w + 255) / 256, a->out_h), 256, 0, st>>>(in, a->out_w, a->dst, row0, a->bounds_v,
                                                                              a->coeffs_v, a->ksize_v);
        GMS_AFTER_LAUNCH("resize_v_u8", 0, st);
    }
    return GMS_OK;
}

int gms_adam_sh_factored(const gms_adam_sh_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->xyz || !a->exchange || !a->p || !a->m || !a->v || a->P < 0 || a->M != 16 || a->R < 1 || a->step < 1 ||
        a->sh_degree < 0 || a->sh_degree > 3 || a->slot_floats < 3 * (int64_t)a->P + 3)
        return set_err(GMS_E_ARG, "gms_adam_sh_factored: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    AdamShArgs k;
    k.P = a->P; k.D = a->sh_degree; k.R = a->R; k.slot = a->slot_floats; k.xyz = a->xyz; k.xbuf = a->exchange;
    k.p = a->p; k.m = a->m; k.v = a->v; k.scale = a->grad_scale;
    k.c = adam_sh_const(a->lr_dc, a->lr_rest, a->beta1, a->beta2, a->eps, a->step);
    span_begin(K_ADAM, st);
    if (g_opt_adam_sh_ieee) k_adam_sh<true><<<(a->P + 127) / 128, 128, 0, st>>>(k);
    else k_adam_sh<false><<<(a->P + 127) / 128, 128, 0, st>>>(k);
    GMS_AFTER_LAUNCH("adam_sh", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_frame_views(void* workspace, int32_t P, int32_t W, int32_t H, gms_frame_view* v) {
    if (!workspace || !v) return set_err(GMS_E_ARG, "gms_frame_views: null argument%s%s");
    FrameLayout FL = frame_layout(aligned_base_c(workspace), P, W, H);
    v->xyz = FL.xyz; v->scales = FL.scales; v->rotations = FL.rots; v->opacities = FL.opac; v->radii = FL.radii;
    v->image = FL.image; v->invdepth = FL.invdepth;
    return GMS_OK;
}

const char* gms_last_error(void) { return g_err; }
const char* gms_version(void) { return "gms_b200 0.1 (sm_90a)"; }
int64_t gms_launch_count(int reset) { const int64_t v = g_launches; if (reset) g_launches = 0; return v; }

int gms_set_option(const char* key, int value) {
    int* p = nullptr;
    if (!strcmp(key, "warp_emit")) p = &g_opt_warp_emit;
    else if (!strcmp(key, "time_kernels")) p = &g_opt_time;
    else if (!strcmp(key, "composite_fwd")) p = &g_opt_fwd;
    else if (!strcmp(key, "composite_bwd")) p = &g_opt_bwd;
    else if (!strcmp(key, "bwd_minblocks")) p = &g_opt_bwd_minb;
    else if (!strcmp(key, "key16")) p = &g_opt_key16;
    else if (!strcmp(key, "adam_sh_ieee")) p = &g_opt_adam_sh_ieee;
    else if (!strcmp(key, "tile_order")) p = &g_opt_tile_order;
    else if (!strcmp(key, "sort_impl")) p = &g_opt_sort;
    else if (!strcmp(key, "bin_impl")) p = &g_opt_bin;
    else if (!strcmp(key, "expand_staged")) p = &g_opt_expand_staged;
    else if (!strcmp(key, "expand_wide")) p = &g_opt_expand_wide;
    else if (!strcmp(key, "sh_staged")) p = &g_opt_sh_staged;
    else if (!strcmp(key, "pre_bwd_minblocks")) p = &g_opt_pre_bwd_minb;
    if (!p) return -1;
    const int old = *p; *p = value; return old;
}

int gms_kernel_times(int reset, int max_kernels, double* ms_out, int64_t* count_out, const char** names_out) {
    spans_collect();
    const int n = max_kernels < K_COUNT ? max_kernels : K_COUNT;
    for (int i = 0; i < n; i++) {
        if (ms_out) ms_out[i] = g_ktime_ms[i];
        if (count_out) count_out[i] = g_kcount[i];
        if (names_out) names_out[i] = g_kernel_names[i];
    }
    if (reset) for (int i = 0; i < K_COUNT; i++) { g_ktime_ms[i] = 0.0; g_kcount[i] = 0; }
    return K_COUNT;
}

int gms_scratch_bytes(int32_t P, int32_t W, int32_t H, size_t* geom_bytes, size_t* image_bytes) {
    if (P < 0 || W <= 0 || H <= 0) return set_err(GMS_E_ARG, "gms_scratch_bytes: bad sizes%s%s");
    if (geom_bytes) *geom_bytes = geom_layout(nullptr, P).total + 256;
    if (image_bytes) *image_bytes = image_layout(nullptr, W, H).total + 256;
    return GMS_OK;
}

size_t gms_binning_bytes(int64_t num_rendered, int32_t P) { (void)P; return bin_layout(nullptr, num_rendered).total_with_lists + 256; }

static int check_inputs(const gms_raster_inputs* in) {
    if (!in || in->P < 0) return set_err(GMS_E_ARG, "bad inputs%s%s");
    if ((in->shs != nullptr) == (in->colors_precomp != nullptr))
        return set_err(GMS_E_ARG, "Please provide excatly one of either SHs or precomputed colors!%s%s");
    const bool sr = in->scales != nullptr || in->rotations != nullptr;
    if ((sr && in->cov3D_precomp) || (!sr && !in->cov3D_precomp) || (sr && (!in->scales || !in->rotations)))
        return set_err(GMS_E_ARG, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!%s%s");
    if (in->shs && (in->M <= 0 || in->M > 16)) return set_err(GMS_E_ARG, "shs must hold 1..16 coefficients per Gaussian%s%s");
    const uintptr_t al = (uintptr_t)in->shs | (uintptr_t)in->rotations | (uintptr_t)in->means3D | (uintptr_t)in->scales |
                         (uintptr_t)in->opacities | (uintptr_t)in->colors_precomp | (uintptr_t)in->cov3D_precomp;
    if (al & 15) return set_err(GMS_E_ARG, "input tensors must be 16-byte aligned (128-bit loads)%s%s");
    return GMS_OK;
}

static PreArgs make_pre_args(const gms_raster_settings* s, const gms_raster_inputs* in) {
    PreArgs a;
    a.P = in->P; a.D = s->sh_degree; a.M = in->M; a.W = s->image_width; a.H = s->image_height;
    a.gx = (a.W + GMS_TILE - 1) / GMS_TILE; a.gy = (a.H + GMS_TILE - 1) / GMS_TILE;
    a.antialiasing = s->antialiasing;
    a.tanfovx = s->tanfovx; a.tanfovy = s->tanfovy;
    a.focal_x = (float)a.W / (2.0f * s->tanfovx); a.focal_y = (float)a.H / (2.0f * s->tanfovy);
    a.mod = s->scale_modifier;
    a.means = in->means3D; a.scales = in->scales; a.rots = in->rotations; a.cov_pre = in->cov3D_precomp;
    a.opac = in->opacities; a.shs = in->shs; a.colors_pre = in->colors_precomp;
    a.opac_raw = nullptr; a.opac_out = nullptr;
    a.view = s->viewmatrix; a.proj = s->projmatrix; a.campos = s->campos;
    return a;
}

static void* aligned_base(void* p) { return reinterpret_cast<void*>(align_up(reinterpret_cast<size_t>(p))); }

// nosync_capacity > 0: never synchronise with the host -- the binning region is requested for that many duplicates, N stays
// on the device (and, when n_host is given, is mirrored into mapped pinned host memory by the kernel that computes it).
static int raster_forward_impl(const gms_raster_settings* s, const gms_raster_inputs* in, const gms_raster_outputs* out,
                               gms_alloc_fn alloc, void* user, gms_raster_saved* saved, void* cuda_stream,
                               int64_t nosync_capacity, uint32_t* n_host, const float* opac_raw = nullptr) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!s || !out || !alloc || !saved || !in) return set_err(GMS_E_ARG, "null argument%s%s");
    int rc = in->P == 0 ? GMS_OK : check_inputs(in);   // P = 0: nothing to check, background-only images (stock behaviour)
    if (rc) return rc;
    if (s->sh_degree < 0 || s->sh_degree > 3) return set_err(GMS_E_UNSUPPORTED, "sh_degree must be 0..3%s%s");
    if (in->shs && (s->sh_degree + 1) * (s->sh_degree + 1) > in->M) return set_err(GMS_E_ARG, "sh_degree needs more coefficients than shs holds%s%s");
    const int P = in->P, W = s->image_width, H = s->image_height;
    const int gx = (W + GMS_TILE - 1) / GMS_TILE, gy = (H + GMS_TILE - 1) / GMS_TILE, T = gx * gy;
    const int dbg = s->debug;
    saved->geom = saved->binning = saved->image = nullptr; saved->num_rendered = 0; saved->num_visible = -1;
    saved->binning_capacity = 0; saved->flags = 0;
    if (g_opt_fwd != 2 && g_opt_fwd != 3) return set_err(GMS_E_ARG, "option composite_fwd must be 2 or 3%s%s");

    size_t gb = 0, ib = 0;
    gms_scratch_bytes(P, W, H, &gb, &ib);
    void* img_raw = alloc(user, GMS_BUF_IMAGE, ib);
    if (!img_raw) return set_err(GMS_E_ALLOC, "image scratch allocation failed%s%s");
    saved->image = img_raw;
    ImageLayout IL = image_layout(aligned_base(img_raw), W, H);
    GMS_CUDA(cudaMemsetAsync(IL.ranges, 0, sizeof(int2) * (size_t)T, st));

    if (P == 0) {   // stock: returns background-only images without launching the pipeline
        const size_t HW = (size_t)W * H;
        k_fill_background<<<(unsigned)((HW + 255) / 256), 256, 0, st>>>(W, H, s->bg, out->out_color, out->out_invdepth);
        GMS_AFTER_LAUNCH("fill_background", dbg, st);
        GMS_CUDA(cudaMemsetAsync(IL.tile_last, 0, sizeof(int) * (size_t)T, st));
        GMS_CUDA(cudaMemsetAsync(IL.n_contrib, 0, sizeof(int) * HW, st));
        return GMS_OK;
    }
    void* geom_raw = alloc(user, GMS_BUF_GEOM, gb);
    if (!geom_raw) return set_err(GMS_E_ALLOC, "geom scratch allocation failed%s%s");
    saved->geom = geom_raw;
    GeomLayout GL = geom_layout(aligned_base(geom_raw), P);

    PreArgs pa = make_pre_args(s, in);
    if (opac_raw) { pa.opac_raw = opac_raw; pa.opac_out = const_cast<float*>(in->opacities); }
    GMS_CUDA(cudaMemsetAsync(GL.counters, 0, 64 * sizeof(uint32_t), st));
    span_begin(K_PRE_FWD, st);
    if (g_opt_sh_staged && pa.shs && pa.M == 16)
        k_preprocess_fwd<true><<<(P + 127) / 128, 128, 0, st>>>(pa, out->radii, GL.rec, GL.cov3D, GL.clamped, GL.tiles, GL.dkey, GL.idx, GL.rect, GL.counters);
    else
        k_preprocess_fwd<false><<<(P + 127) / 128, 128, 0, st>>>(pa, out->radii, GL.rec, GL.cov3D, GL.clamped, GL.tiles, GL.dkey, GL.idx, GL.rect, GL.counters);
    GMS_AFTER_LAUNCH("preprocess_fwd", dbg, st);
    span_end(st);

    // Tile binning by the cooperative counting kernel (default) when its shared-memory rows fit: needs the depth order only.
    const size_t bin_smem = gms_bin_smem_bytes(T);
    int bin_ctas = 0;       // co-resident CTAs per SM of the cooperative binning kernel (0: its shared-memory rows do not fit)
    sm_count();
    if (g_opt_bin && bin_smem + 12288 <= (size_t)g_bin_smem_optin && gx < 65536 && gy < 65536) {
        static size_t cached_smem = 0; static int cached_ctas = 0;
        if (cached_smem != bin_smem) {
            GMS_CUDA(cudaFuncSetAttribute(k_bin_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bin_smem));
            GMS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cached_ctas, k_bin_tiles, GMS_BIN_THREADS, bin_smem));
            cached_smem = bin_smem;
        }
        bin_ctas = cached_ctas > 2 ? 2 : cached_ctas;
    }
    const int G = bin_ctas * sm_count();
    const bool counting = bin_ctas >= 1;
    if (!g_pinned) GMS_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&g_pinned), 64, cudaHostAllocDefault));
    cudaEvent_t n_ready = nullptr;
    if (counting && nosync_capacity <= 0) {     // stock-compatible call: N (= sum of tiles_touched) sizes the binning region
        GMS_CUDA(cudaMemcpyAsync(g_pinned, GL.counters + 3, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        GMS_CUDA(cudaEventCreateWithFlags(&n_ready, cudaEventDisableTiming));
        GMS_CUDA(cudaEventRecord(n_ready, st));   // waited for AFTER the depth sort has been queued
    }

    // depth order of the P Gaussians (stable => ties keep ascending index), then offsets in that order
    size_t tb = GL.cub_bytes;
    const uint32_t* order = GL.order;
    span_begin(K_SORT_P, st);
    if (g_opt_sort) {
        k_set_u32<<<1, 1, 0, st>>>(GL.counters + 1, (uint32_t)P);
        const int res = gms_radix_sort_pairs(GL.dkey, nullptr, GL.dkey_s, GL.order, GL.dkey_t, GL.order_t, GL.counters + 1, P, 32,
                                             GL.sort_temp, st, &g_launches);
        if (res < 0) return set_err(GMS_E_CUDA, "radix sort (depth) launch failed%s%s");
        order = res ? GL.order_t : GL.order;
    } else {
        GMS_CUDA(cub::DeviceRadixSort::SortPairs(GL.cub_temp, tb, GL.dkey, GL.dkey_s, GL.idx, GL.order, P, 0, 32, st));
    }
    span_end(st);
    if (counting) {
        int64_t N = -1, cap = nosync_capacity;
        if (n_ready) {
            const cudaError_t e = cudaEventSynchronize(n_ready);
            cudaEventDestroy(n_ready);
            if (e != cudaSuccess) return set_err(GMS_E_CUDA, "waiting for N: %s", cudaGetErrorString(e));
            N = (int64_t)g_pinned[0];
            cap = N;
        }
        saved->num_rendered = N;
        saved->flags = 1;
        saved->binning_capacity = cap;
        if (cap > 0) {
            // binning region: the point list, then (unless this is a forward-only call) the per-quad survivor lists
            const bool emit = !(out->flags & GMS_FORWARD_ONLY) && g_opt_fwd == 2 && g_opt_bwd == 5;
            const size_t pl_bytes = align_up((size_t)cap * sizeof(uint32_t));
            void* bin_raw = alloc(user, GMS_BUF_BINNING, pl_bytes * (emit ? 5 : 1) + 256);
            if (!bin_raw) return set_err(GMS_E_ALLOC, "binning scratch allocation failed%s%s");
            saved->binning = bin_raw;
            uint32_t* point_list = reinterpret_cast<uint32_t*>(aligned_base(bin_raw));
            uint32_t* surv = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(point_list) + pl_bytes);
            if (emit) saved->flags |= 2;
            GmsBinArgs ba;
            ba.P = P; ba.T = T; ba.gx = gx; ba.order = order; ba.rect = GL.rect; ba.nvis = GL.counters + 2;
            ba.M = IL.binM; ba.total = IL.bin_total; ba.ranges = IL.ranges; ba.point_list = point_list; ba.tile_keys = nullptr;
            ba.capacity = (uint32_t)(cap > 0xFFFFFFFFll ? 0xFFFFFFFFll : cap); ba.n_out = GL.counters; ba.n_host = n_host;
            void* kargs[] = {&ba};
            span_begin(K_SORT_N, st);
            GMS_CUDA(cudaLaunchCooperativeKernel((void*)k_bin_tiles, dim3(G), dim3(GMS_BIN_THREADS), kargs, bin_smem, st));
            GMS_AFTER_LAUNCH("bin_tiles", dbg, st);
            span_end(st);
            if (g_opt_tile_order) {
                k_tile_order<<<1, 1024, 0, st>>>(T, IL.ranges, IL.tile_order);
                GMS_AFTER_LAUNCH("tile_order", dbg, st);
            }
            span_begin(K_COMP_FWD, st);
            if (g_opt_fwd == 3)
                k_composite_fwd3<<<T, GMS_CB, 0, st>>>(IL.ranges, g_opt_tile_order ? IL.tile_order : nullptr, point_list, GL.rec, W, H, gx, s->bg,
                                                      out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth);
            else if (emit)
                k_composite_fwd2<true><<<T, GMS_CB, 0, st>>>(IL.ranges, g_opt_tile_order ? IL.tile_order : nullptr, point_list, GL.rec, W, H, gx, s->bg,
                                                            out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth, surv, IL.nsurv);
            else
                k_composite_fwd2<false><<<T, GMS_CB, 0, st>>>(IL.ranges, g_opt_tile_order ? IL.tile_order : nullptr, point_list, GL.rec, W, H, gx, s->bg,
                                                             out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth, nullptr, nullptr);
            GMS_AFTER_LAUNCH("composite_fwd", dbg, st);
            span_end(st);
        } else {
            const size_t HW = (size_t)W * H;
            k_fill_background<<<(unsigned)((HW + 255) / 256), 256, 0, st>>>(W, H, s->bg, out->out_color, out->out_invdepth);
            GMS_AFTER_LAUNCH("fill_background", dbg, st);
            GMS_CUDA(cudaMemsetAsync(IL.n_contrib, 0, sizeof(int) * HW, st));
        }
        return GMS_OK;
    }
    {
        auto it = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), TilesInOrder{GL.tiles, order});
        tb = GL.cub_bytes;
        span_begin(K_SCAN, st);
        GMS_CUDA(cub::DeviceScan::InclusiveSum(GL.cub_temp, tb, it, GL.offs, P, st));
        span_end(st);
    }
    // N = offs[P-1] stays on the device.  Stock-style call: one 4-byte read-back sizes the binning region exactly (cap = N).
    // Sync-free call: the region is sized for `nosync_capacity` entries, the tail beyond N is filled with sentinel keys that
    // sort behind every tile, and the sort runs over the whole capacity.
    int64_t N = -1, cap = nosync_capacity;
    if (nosync_capacity <= 0) {
        GMS_CUDA(cudaMemcpyAsync(g_pinned, GL.offs + (P - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        GMS_CUDA(cudaStreamSynchronize(st));
        N = (int64_t)g_pinned[0];
        cap = N;
    }
    saved->num_rendered = N;
    saved->binning_capacity = cap;

    if (cap > 0) {
        const bool emit = !(out->flags & GMS_FORWARD_ONLY) && g_opt_fwd == 2 && g_opt_bwd == 5;
        BinLayout BL = bin_layout(nullptr, cap);
        void* bin_raw = alloc(user, GMS_BUF_BINNING, (emit ? BL.total_with_lists : BL.total) + 256);
        if (!bin_raw) return set_err(GMS_E_ALLOC, "binning scratch allocation failed%s%s");
        saved->binning = bin_raw;
        if (emit) saved->flags |= 2;
        BL = bin_layout(aligned_base(bin_raw), cap);
        const int tbits = gms_tile_bits((uint32_t)T);
        const int npass = (tbits + 7) / 8;
        // hand-written sort ping-pongs between the two key/value pairs: emit into the one that makes the LAST pass land in
        // (keys_out, vals_out), which is where every later kernel (and backward) expects the sorted list
        const bool emit_into_out = g_opt_sort && (npass % 2 == 0);
        uint32_t* ek = emit_into_out ? BL.keys_out : BL.keys_in;
        uint32_t* ev = emit_into_out ? BL.vals_out : BL.vals_in;
        // 16-bit tile keys whenever the tile ids (and the all-ones sentinel behind them) fit: a quarter less traffic through
        // the two sort passes.  The key arrays keep their 32-bit footprint; the hand-written sort stays on 32-bit keys.
        const bool k16 = !g_opt_sort && g_opt_key16 && T <= 65535;
        if (k16) saved->flags |= 4;
        const uint32_t cap32 = (uint32_t)(cap > 0xFFFFFFFFll ? 0xFFFFFFFFll : cap);
        // Sync-free call: sentinel keys behind the N emitted ones, written BEFORE the emit.  cub sorts the whole capacity, so
        // they go into its input (ek).  The hand-written sort moves only the N device-side items and leaves the tail of every
        // buffer as it was, so they go into its final output, keys_out -- which is also the emit target when the sort takes
        // an even number of passes, so nothing may write keys_out between the emit and the sort.
        if (N < 0) GMS_CUDA(cudaMemsetAsync(g_opt_sort ? BL.keys_out : ek, 0xFF, (k16 ? sizeof(uint16_t) : sizeof(uint32_t)) * (size_t)cap, st));
        span_begin(K_EMIT, st);
        if (k16) k_emit_dups<uint16_t><<<(P + 255) / 256, 256, 0, st>>>(P, gx, order, GL.offs, GL.rect, reinterpret_cast<uint16_t*>(ek), ev, g_opt_warp_emit, cap32);
        else k_emit_dups<uint32_t><<<(P + 255) / 256, 256, 0, st>>>(P, gx, order, GL.offs, GL.rect, ek, ev, g_opt_warp_emit, cap32);
        GMS_AFTER_LAUNCH("emit_dups", dbg, st);
        span_end(st);
        size_t sb = BL.cub_bytes;
        span_begin(K_SORT_N, st);
        if (g_opt_sort) {
            uint32_t* k0 = emit_into_out ? BL.keys_in : BL.keys_out; uint32_t* v0 = emit_into_out ? BL.vals_in : BL.vals_out;
            uint32_t* k1 = emit_into_out ? BL.keys_out : BL.keys_in; uint32_t* v1 = emit_into_out ? BL.vals_out : BL.vals_in;
            const int res = gms_radix_sort_pairs(ek, ev, k0, v0, k1, v1, GL.offs + (P - 1), cap, tbits, BL.sort_temp, st, &g_launches);
            if (res < 0 || (res ? k1 : k0) != BL.keys_out) return set_err(GMS_E_CUDA, "radix sort (tiles) failed%s%s");
        } else if (k16) {
            GMS_CUDA(cub::DeviceRadixSort::SortPairs(BL.cub_temp, sb, reinterpret_cast<uint16_t*>(BL.keys_in), reinterpret_cast<uint16_t*>(BL.keys_out),
                                                     BL.vals_in, BL.vals_out, (int)cap, 0, tbits, st));
        } else {
            GMS_CUDA(cub::DeviceRadixSort::SortPairs(BL.cub_temp, sb, BL.keys_in, BL.keys_out, BL.vals_in, BL.vals_out, (int)cap, 0, tbits, st));
        }
        span_end(st);
        span_begin(K_RANGES, st);
        if (k16) k_tile_ranges<uint16_t><<<(unsigned)((cap + 255) / 256), 256, 0, st>>>(cap, reinterpret_cast<const uint16_t*>(BL.keys_out), IL.ranges, (uint32_t)T,
                                                                                        GL.offs + (P - 1), GL.counters, n_host);
        else k_tile_ranges<uint32_t><<<(unsigned)((cap + 255) / 256), 256, 0, st>>>(cap, BL.keys_out, IL.ranges, (uint32_t)T, GL.offs + (P - 1), GL.counters, n_host);
        GMS_AFTER_LAUNCH("tile_ranges", dbg, st);
        span_end(st);
        if (g_opt_tile_order) {
            k_tile_order<<<1, 1024, 0, st>>>(T, IL.ranges, IL.tile_order);
            GMS_AFTER_LAUNCH("tile_order", dbg, st);
        }
        span_begin(K_COMP_FWD, st);
        if (g_opt_fwd == 3)
            k_composite_fwd3<<<T, GMS_CB, 0, st>>>(IL.ranges, g_opt_tile_order ? IL.tile_order : nullptr, BL.vals_out, GL.rec, W, H, gx, s->bg,
                                                  out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth);
        else if (emit)
            k_composite_fwd2<true><<<T, GMS_CB, 0, st>>>(IL.ranges, g_opt_tile_order ? IL.tile_order : nullptr, BL.vals_out, GL.rec, W, H, gx, s->bg,
                                                        out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth, BL.surv, IL.nsurv);
        else
            k_composite_fwd2<false><<<T, GMS_CB, 0, st>>>(IL.ranges, g_opt_tile_order ? IL.tile_order : nullptr, BL.vals_out, GL.rec, W, H, gx, s->bg,
                                                         out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth, nullptr, nullptr);
        GMS_AFTER_LAUNCH("composite_fwd", dbg, st);
        span_end(st);
    } else {
        const size_t HW = (size_t)W * H;
        k_fill_background<<<(unsigned)((HW + 255) / 256), 256, 0, st>>>(W, H, s->bg, out->out_color, out->out_invdepth);
        GMS_AFTER_LAUNCH("fill_background", dbg, st);
        GMS_CUDA(cudaMemsetAsync(IL.tile_last, 0, sizeof(int) * (size_t)T, st));
        GMS_CUDA(cudaMemsetAsync(IL.n_contrib, 0, sizeof(int) * HW, st));
    }
    return GMS_OK;
}

int gms_rasterize_forward(const gms_raster_settings* s, const gms_raster_inputs* in, const gms_raster_outputs* out,
                          gms_alloc_fn alloc, void* user, gms_raster_saved* saved, void* cuda_stream) {
    return raster_forward_impl(s, in, out, alloc, user, saved, cuda_stream, 0, nullptr);
}

int gms_rasterize_forward_nosync(const gms_raster_settings* s, const gms_raster_inputs* in, const gms_raster_outputs* out,
                                 gms_alloc_fn alloc, void* user, gms_raster_saved* saved, int64_t binning_capacity,
                                 uint32_t* n_host_mapped, void* cuda_stream) {
    if (binning_capacity <= 0) return set_err(GMS_E_ARG, "gms_rasterize_forward_nosync: binning_capacity must be > 0%s%s");
    return raster_forward_impl(s, in, out, alloc, user, saved, cuda_stream, binning_capacity, n_host_mapped);
}

static int raster_backward_impl(const gms_raster_settings* s, const gms_raster_inputs* in, const int32_t* radii,
                                const gms_raster_saved* saved, const float* dL_dout_color, const float* dL_dout_invdepth,
                                const gms_raster_grads* gr, void* cuda_stream, float* dopac_raw, const gms_sh_adam* sh_adam) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!s || !saved || !gr || !dL_dout_color || !in) return set_err(GMS_E_ARG, "null argument%s%s");
    if (in->P == 0) return GMS_OK;
    int rc = check_inputs(in);
    if (rc) return rc;
    const int P = in->P, W = s->image_width, H = s->image_height;
    if (!gr->dL_dmeans3D || !gr->dL_dmeans2D || (!gr->dL_dopacities && !dopac_raw)) return set_err(GMS_E_ARG, "dL_dmeans3D/dL_dmeans2D/dL_dopacities are required%s%s");
    if (!saved->geom || !saved->image) return set_err(GMS_E_ARG, "saved scratch missing%s%s");
    const int gx = (W + GMS_TILE - 1) / GMS_TILE, gy = (H + GMS_TILE - 1) / GMS_TILE, T = gx * gy;
    const int dbg = s->debug;
    GeomLayout GL = geom_layout(aligned_base(saved->geom), P);
    ImageLayout IL = image_layout(aligned_base(saved->image), W, H);
    GMS_CUDA(cudaMemsetAsync(GL.dgeom, 0, sizeof(float4) * 3 * (size_t)P, st));
    const bool counting = (saved->flags & 1) != 0;        // binning region = the point list (+ survivor lists) alone (gms_binning.cuh)
    if (saved->binning_capacity > 0) {
        if (!saved->binning) return set_err(GMS_E_ARG, "saved binning scratch missing%s%s");
        BinLayout BL = bin_layout(aligned_base(saved->binning), counting ? 1 : saved->binning_capacity);
        if (counting) BL.vals_out = reinterpret_cast<uint32_t*>(aligned_base(saved->binning));
        span_begin(K_COMP_BWD, st);
        {
            const int* to = g_opt_tile_order ? IL.tile_order : nullptr;
            const bool depth = dL_dout_invdepth != nullptr;
            const bool lists = (saved->flags & 2) != 0;       // the forward wrote per-quad survivor lists
            const uint32_t* surv = !lists ? nullptr : !counting ? BL.surv :
                reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(BL.vals_out) + align_up((size_t)saved->binning_capacity * sizeof(uint32_t)));
#define GMS_BWD_ARGS IL.ranges, to, BL.vals_out, GL.rec, W, H, gx, s->bg, IL.final_T, IL.n_contrib, dL_dout_color, dL_dout_invdepth, GL.dgeom
#define GMS_BWD_LAUNCH(MB)                                                                                                        \
            do {                                                                                                                  \
                if (lists) { if (depth) k_composite_bwd5<MB, true><<<T, GMS_CB, 0, st>>>(GMS_BWD_ARGS, surv, IL.nsurv);           \
                             else k_composite_bwd5<MB, false><<<T, GMS_CB, 0, st>>>(GMS_BWD_ARGS, surv, IL.nsurv); }              \
                else { if (depth) k_composite_bwd3<MB, true><<<T, GMS_CB, 0, st>>>(GMS_BWD_ARGS);                                 \
                       else k_composite_bwd3<MB, false><<<T, GMS_CB, 0, st>>>(GMS_BWD_ARGS); }                                    \
            } while (0)
            if (g_opt_bwd_minb >= 8) GMS_BWD_LAUNCH(8);
            else if (g_opt_bwd_minb >= 6) GMS_BWD_LAUNCH(6);
            else if (g_opt_bwd_minb == 5) GMS_BWD_LAUNCH(5);
            else GMS_BWD_LAUNCH(4);
#undef GMS_BWD_LAUNCH
#undef GMS_BWD_ARGS
        }
        GMS_AFTER_LAUNCH("composite_bwd", dbg, st);
        span_end(st);
    }
    PreBwdArgs b;
    b.f = make_pre_args(s, in);
    b.radii = radii; b.cov3D = GL.cov3D; b.clamped = GL.clamped; b.dgeom = GL.dgeom;
    b.dmeans3D = gr->dL_dmeans3D; b.dmeans2D = gr->dL_dmeans2D; b.dopac = gr->dL_dopacities;
    b.dshs = in->shs ? gr->dL_dshs : nullptr;
    b.dcolors_pre = in->colors_precomp ? gr->dL_dcolors_precomp : nullptr;
    b.dscales = in->scales ? gr->dL_dscales : nullptr;
    b.drots = in->rotations ? gr->dL_drotations : nullptr;
    b.dcov_pre = in->cov3D_precomp ? gr->dL_dcov3D_precomp : nullptr;
    b.dcol_sh = in->shs ? gr->dL_dcolors_sh : nullptr;
    b.dopac_raw = dopac_raw;
    span_begin(K_PRE_BWD, st);
    if (sh_adam) {          // factored SH gradient applied in place: the SH Adam step of the frame (gms_sh_adam)
        if (b.f.M != 16 || !b.f.shs) return set_err(GMS_E_ARG, "sh_adam needs shs with 16 coefficients%s%s");
        b.dshs = nullptr;
        b.sh_p = const_cast<float*>(b.f.shs); b.sh_m = sh_adam->m; b.sh_v = sh_adam->v;
        b.sh_adam = adam_sh_const(sh_adam->lr_dc, sh_adam->lr_rest, sh_adam->beta1, sh_adam->beta2, sh_adam->eps, sh_adam->step);
        const int grid = (P + 127) / 128;
        if (g_opt_pre_bwd_minb >= 4) {
            if (g_opt_adam_sh_ieee) k_preprocess_bwd<1, 4, true, true, true><<<grid, 128, 0, st>>>(b);
            else k_preprocess_bwd<1, 4, true, true><<<grid, 128, 0, st>>>(b);
        } else {
            if (g_opt_adam_sh_ieee) k_preprocess_bwd<1, 1, true, true, true><<<grid, 128, 0, st>>>(b);
            else k_preprocess_bwd<1, 1, true, true><<<grid, 128, 0, st>>>(b);
        }
    } else if (b.dcol_sh) {        // factored SH gradient
        if (b.f.M != 16 || !b.f.shs) return set_err(GMS_E_ARG, "dL_dcolors_sh needs shs with 16 coefficients%s%s");
        b.dshs = nullptr;
        if (g_opt_pre_bwd_minb >= 4) k_preprocess_bwd<1, 4, true><<<(P + 127) / 128, 128, 0, st>>>(b);
        else k_preprocess_bwd<1, 1, true><<<(P + 127) / 128, 128, 0, st>>>(b);
    } else if (g_opt_sh_staged && b.f.shs && b.dshs && b.f.M == 16) {
        const int grid = (P + 127) / 128;
        if (g_opt_sh_staged == 2) {
            if (g_opt_pre_bwd_minb >= 4) k_preprocess_bwd<2, 4><<<grid, 128, 0, st>>>(b);
            else k_preprocess_bwd<2, 1><<<grid, 128, 0, st>>>(b);
        } else {
            if (g_opt_pre_bwd_minb >= 4) k_preprocess_bwd<1, 4><<<grid, 128, 0, st>>>(b);
            else k_preprocess_bwd<1, 1><<<grid, 128, 0, st>>>(b);
        }
    } else k_preprocess_bwd<0, 1><<<(P + 127) / 128, 128, 0, st>>>(b);
    GMS_AFTER_LAUNCH("preprocess_bwd", dbg, st);
    span_end(st);
    return GMS_OK;
}

int gms_rasterize_backward(const gms_raster_settings* s, const gms_raster_inputs* in, const int32_t* radii,
                           const gms_raster_saved* saved, const float* dL_dout_color, const float* dL_dout_invdepth,
                           const gms_raster_grads* gr, void* cuda_stream) {
    return raster_backward_impl(s, in, radii, saved, dL_dout_color, dL_dout_invdepth, gr, cuda_stream, nullptr, nullptr);
}

int gms_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present, void* cuda_stream) {
    (void)projmatrix;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (P <= 0) return GMS_OK;
    k_mark_visible<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, viewmatrix, present);
    GMS_AFTER_LAUNCH("mark_visible", 0, st);
    return GMS_OK;
}

int gms_debug_get_views(const gms_raster_saved* saved, int32_t P, int32_t W, int32_t H, gms_debug_views* v) {
    if (!saved || !v) return set_err(GMS_E_ARG, "null argument%s%s");
    memset(v, 0, sizeof(*v));
    if (saved->geom) {
        GeomLayout GL = geom_layout(aligned_base(saved->geom), P);
        v->cov3D = GL.cov3D; v->tiles_touched = GL.tiles;
        v->means2D = reinterpret_cast<const float*>(GL.rec);   // packed records; use gms_debug_unpack for stock layouts
    }
    if (saved->image) {
        ImageLayout IL = image_layout(aligned_base(saved->image), W, H);
        v->final_T = IL.final_T; v->n_contrib = IL.n_contrib; v->ranges = reinterpret_cast<const int32_t*>(IL.ranges);
        if (saved->geom) v->dgeom = reinterpret_cast<const float*>(geom_layout(aligned_base(saved->geom), P).dgeom);
    }
    if (saved->binning && (saved->flags & 1)) {
        v->point_list = reinterpret_cast<const uint32_t*>(aligned_base(saved->binning)); v->tile_keys = nullptr;
    } else if (saved->binning && saved->binning_capacity > 0) {
        BinLayout BL = bin_layout(aligned_base(saved->binning), saved->binning_capacity);
        v->point_list = BL.vals_out; v->tile_keys = (saved->flags & 4) ? nullptr : BL.keys_out;     // (16-bit keys: callers derive them from the ranges)
    }
    return GMS_OK;
}

int gms_debug_unpack(const gms_raster_saved* saved, int32_t P, const int32_t* radii, float* means2D, float* depths,
                     float* conic_opacity, float* rgb, uint8_t* clamped, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!saved || !saved->geom || P <= 0) return set_err(GMS_E_ARG, "nothing to unpack%s%s");
    GeomLayout GL = geom_layout(aligned_base(saved->geom), P);
    k_unpack<<<(P + 255) / 256, 256, 0, st>>>(P, GL.rec, GL.clamped, GL.dkey, radii, means2D, depths, conic_opacity, rgb, clamped);
    GMS_AFTER_LAUNCH("unpack", 0, st);
    return GMS_OK;
}

// Which expansion kernels a call runs: the warp-per-face ones (option "expand_wide") or the per-thread ones.
static bool expand_wide(const gms_expand_args& a) {
    return g_opt_expand_wide == 2 || (g_opt_expand_wide == 1 && a.alpha_activation == GMS_ALPHA_SOFTMAX && a.K >= GMS_EXP_WIDE_MIN_K);
}

int gms_expand_forward(const gms_expand_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->F < 0 || a->K <= 0) return set_err(GMS_E_ARG, "bad expansion sizes%s%s");
    if (!a->triangles_in && (!a->vertices || !a->faces)) return set_err(GMS_E_ARG, "vertices/faces or triangles_in required%s%s");
    if (!a->alpha_raw || !a->scale_raw) return set_err(GMS_E_ARG, "_alpha and _scale required%s%s");
    if (a->alpha_activation != GMS_ALPHA_RELU && a->alpha_activation != GMS_ALPHA_SOFTMAX)
        return set_err(GMS_E_ARG, "alpha_activation must be 0 (relu) or 1 (softmax)%s%s");
    if (a->F == 0) return GMS_OK;
    span_begin(K_EXP_FWD, st);
    const bool softmax = a->alpha_activation == GMS_ALPHA_SOFTMAX;
    if (expand_wide(*a)) {
        const int grid = (a->F + GMS_EXP_WIDE_BLOCK / 32 - 1) / (GMS_EXP_WIDE_BLOCK / 32);
        if (softmax) k_expand_wide_fwd<GMS_ALPHA_SOFTMAX><<<grid, GMS_EXP_WIDE_BLOCK, 0, st>>>(*a);
        else k_expand_wide_fwd<GMS_ALPHA_RELU><<<grid, GMS_EXP_WIDE_BLOCK, 0, st>>>(*a);
    } else {
        const int grid = (a->F + GMS_EXP_BLOCK - 1) / GMS_EXP_BLOCK;
        const size_t smem = (size_t)GMS_EXP_BLOCK * a->K * exp_fwd_stage_width(*a) * sizeof(float);
        const bool staged = (g_opt_expand_staged & 1) && smem <= 48 * 1024;
        if (softmax) {
            if (staged) k_expand_softmax_fwd<true><<<grid, GMS_EXP_BLOCK, smem, st>>>(*a);
            else k_expand_softmax_fwd<false><<<grid, GMS_EXP_BLOCK, 0, st>>>(*a);
        } else if (staged) k_expand_fwd<true><<<grid, GMS_EXP_BLOCK, smem, st>>>(*a);
        else k_expand_fwd<false><<<grid, GMS_EXP_BLOCK, 0, st>>>(*a);
    }
    GMS_AFTER_LAUNCH("expand_fwd", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_points_expand_forward(const gms_points_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->P < 0 || !a->triangles) return set_err(GMS_E_ARG, "gms_points_expand_forward: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    span_begin(K_EXP_FWD, st);
    k_points_expand_fwd<<<(a->P + 127) / 128, 128, 0, st>>>(*a);
    GMS_AFTER_LAUNCH("points_expand_fwd", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_points_prepare_vertices(const gms_points_vertices_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->P < 0 || (a->scaling_cols != 2 && a->scaling_cols != 3))
        return set_err(GMS_E_ARG, "gms_points_prepare_vertices: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    if (!a->xyz || !a->scaling_log || !a->rotation_raw || !a->triangles)
        return set_err(GMS_E_ARG, "gms_points_prepare_vertices: null buffer%s%s");
    span_begin(K_EXP_FWD, st);
    k_points_vertices<<<(a->P + 127) / 128, 128, 0, st>>>(*a);
    GMS_AFTER_LAUNCH("points_vertices", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_expand_backward(const gms_expand_args* a, const gms_expand_grads* g, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !g || a->F < 0 || a->K <= 0) return set_err(GMS_E_ARG, "bad expansion sizes%s%s");
    if (!a->triangles_in && (!a->vertices || !a->faces)) return set_err(GMS_E_ARG, "vertices/faces or triangles_in required%s%s");
    if (!a->alpha_raw || !a->scale_raw) return set_err(GMS_E_ARG, "_alpha and _scale required%s%s");
    if (a->alpha_activation != GMS_ALPHA_RELU && a->alpha_activation != GMS_ALPHA_SOFTMAX)
        return set_err(GMS_E_ARG, "alpha_activation must be 0 (relu) or 1 (softmax)%s%s");
    if (a->F == 0) return GMS_OK;
    span_begin(K_EXP_BWD, st);
    const bool softmax = a->alpha_activation == GMS_ALPHA_SOFTMAX;
    if (expand_wide(*a)) {
        const int grid = (a->F + GMS_EXP_WIDE_BLOCK / 32 - 1) / (GMS_EXP_WIDE_BLOCK / 32);
        if (softmax) k_expand_wide_bwd<GMS_ALPHA_SOFTMAX><<<grid, GMS_EXP_WIDE_BLOCK, 0, st>>>(*a, *g);
        else k_expand_wide_bwd<GMS_ALPHA_RELU><<<grid, GMS_EXP_WIDE_BLOCK, 0, st>>>(*a, *g);
    } else {
        const int grid = (a->F + GMS_EXP_BLOCK - 1) / GMS_EXP_BLOCK;
        const size_t smem = (size_t)GMS_EXP_BLOCK * a->K * exp_bwd_stage_width(*g) * sizeof(float);
        const bool staged = (g_opt_expand_staged & 2) && smem <= 48 * 1024;
        if (softmax) {
            if (staged) k_expand_softmax_bwd<true><<<grid, GMS_EXP_BLOCK, smem, st>>>(*a, *g);
            else k_expand_softmax_bwd<false><<<grid, GMS_EXP_BLOCK, 0, st>>>(*a, *g);
        } else if (staged) k_expand_bwd<true><<<grid, GMS_EXP_BLOCK, smem, st>>>(*a, *g);
        else k_expand_bwd<false><<<grid, GMS_EXP_BLOCK, 0, st>>>(*a, *g);
    }
    GMS_AFTER_LAUNCH("expand_bwd", 0, st);
    span_end(st);
    return GMS_OK;
}


size_t gms_frame_workspace_bytes(int32_t P, int32_t W, int32_t H) { return frame_layout(nullptr, P, W, H).total + 512; }

// A whole frame's forward is the model's own expansion step followed by one rasterizer forward, frame_raster_forward, which
// gms_train_frame, gms_render_frame and gms_points_render_frame share.  The expansion writes activated Gaussians (xyz,
// scales, unit quaternions) into the frame's workspace.
struct FrameModel {
    int32_t V, F, K, M;
    const float* vertices; const int64_t* faces; const float* alpha_raw; const float* scale_raw; const float* features;
    const float* opacity_raw; float eps;
    const gms_mesh_segment* segments; int32_t n_segments;
    int32_t alpha_activation;
};

// The Gaussian count of a frame: F*K for one mesh, sum F_i*K_i for a segmented model (gms_mesh_segment), whose sizes are
// validated here, before the frame issues any launch.
static int frame_gaussian_count(const char* fn, const FrameModel& m, int* P) {
    if (m.alpha_activation != GMS_ALPHA_RELU && m.alpha_activation != GMS_ALPHA_SOFTMAX)
        return set_err(GMS_E_ARG, "%s: alpha_activation must be 0 (relu) or 1 (softmax)%s", fn);
    if (m.n_segments == 0) {
        *P = m.F * m.K;
        return GMS_OK;
    }
    if (m.n_segments < 0 || !m.segments) return set_err(GMS_E_ARG, "%s: n_segments < 0, or segments NULL with n_segments > 0%s", fn);
    if (m.K != 0) return set_err(GMS_E_ARG, "%s: K must be 0 when segments are given%s", fn);
    int64_t F = 0, n = 0;
    for (int i = 0; i < m.n_segments; ++i) {
        if (m.segments[i].F < 1 || m.segments[i].K < 1) return set_err(GMS_E_ARG, "%s: every segment needs F >= 1 and K >= 1%s", fn);
        F += m.segments[i].F;
        n += (int64_t)m.segments[i].F * m.segments[i].K;
    }
    if (F != m.F) return set_err(GMS_E_ARG, "%s: F must equal the sum of the segments' F%s", fn);
    if (n > INT32_MAX) return set_err(GMS_E_ARG, "%s: sum of F_i * K_i over the segments exceeds int32%s", fn);
    *P = (int)n;
    return GMS_OK;
}

// gs_mesh: E1-E4 mesh -> Gaussians (activated scales / rotations) into xyz / scales / rots, one launch per mesh segment
// (one in all without segments).  `ea` receives each launch's arguments for the training frame's expansion backward.
static int mesh_expand_forward(const FrameModel& m, float* xyz, float* scales, float* rots, void* cuda_stream,
                               std::vector<gms_expand_args>* ea) {
    const gms_mesh_segment whole = {m.F, m.K};
    const gms_mesh_segment* seg = m.n_segments ? m.segments : &whole;
    const int n = m.n_segments ? m.n_segments : 1;
    ea->assign(n, gms_expand_args());
    size_t f0 = 0, g0 = 0;      // first face and first Gaussian of the segment
    for (int i = 0; i < n; ++i) {
        gms_expand_args& e = (*ea)[i];
        memset(&e, 0, sizeof(e));
        e.V = m.V; e.F = seg[i].F; e.K = seg[i].K; e.vertices = m.vertices; e.faces = m.faces + 3 * f0;
        e.alpha_raw = m.alpha_raw + 3 * g0; e.scale_raw = m.scale_raw + g0; e.eps = m.eps;
        e.xyz = xyz + 3 * g0; e.scaling_act = scales + 3 * g0; e.rotation_act = rots + 4 * g0;
        e.alpha_activation = m.alpha_activation;
        int rc;
        if ((rc = gms_expand_forward(&e, cuda_stream))) return rc;
        f0 += (size_t)seg[i].F;
        g0 += (size_t)seg[i].F * seg[i].K;
    }
    return GMS_OK;
}

// The expansion backward of mesh_expand_forward's launches: per segment, the incoming gradients and the raw-parameter
// gradients are offset like the forward's outputs and inputs; the vertex gradient is shared (accumulated with atomics).
static int mesh_expand_backward(const std::vector<gms_expand_args>& ea, const float* d_xyz, const float* d_scales, const float* d_rots,
                                float* d_vertices, float* d_alpha_raw, float* d_scale_raw, void* cuda_stream) {
    size_t g0 = 0;
    for (const gms_expand_args& e : ea) {
        gms_expand_grads g;
        memset(&g, 0, sizeof(g));
        g.dL_dxyz = d_xyz + 3 * g0; g.dL_dscaling_act = d_scales + 3 * g0; g.dL_drotation_act = d_rots + 4 * g0;
        g.dL_dvertices = d_vertices; g.dL_dalpha_raw = d_alpha_raw + 3 * g0; g.dL_dscale_raw = d_scale_raw + g0;
        int rc;
        if ((rc = gms_expand_backward(&e, &g, cuda_stream))) return rc;
        g0 += (size_t)e.F * e.K;
    }
    return GMS_OK;
}

// The activated Gaussians an expansion step left in the workspace, with the model's SH features and opacity logits.
struct FrameGaussians {
    int32_t P, M;
    const float* xyz; const float* scales; const float* rots; const float* features; const float* opacity_raw;
    float* opac;        // [P] sigmoid(opacity_raw), written by the preprocess for the training frame's backward
};

// The rasterizer forward of a whole frame.  sigmoid(opacity) is computed inside k_preprocess_fwd (which stores it to `opac`),
// its derivative inside k_preprocess_bwd: no separate activation launches.  `in` is filled for the training frame's backward.
static int frame_raster_forward(const FrameGaussians& g, const gms_raster_settings* s, gms_raster_outputs* out, gms_alloc_fn alloc,
                                void* user, int64_t binning_capacity, uint32_t* n_host, void* cuda_stream, gms_raster_inputs* in,
                                gms_raster_saved* saved) {
    memset(in, 0, sizeof(*in));
    in->P = g.P; in->M = g.M; in->means3D = g.xyz; in->opacities = g.opac; in->shs = g.features; in->scales = g.scales;
    in->rotations = g.rots;
    return raster_forward_impl(s, in, out, alloc, user, saved, cuda_stream, binning_capacity, n_host, g.opacity_raw);
}

struct RenderLayout { float* xyz; float* scales; float* rots; float* opac; size_t total; };

static RenderLayout render_layout(void* base, int P) {
    RenderLayout L;
    char* p = reinterpret_cast<char*>(base);
    const size_t Pn = (size_t)(P > 0 ? P : 1);
    L.xyz = carve<float>(p, 3 * Pn); L.scales = carve<float>(p, 3 * Pn); L.rots = carve<float>(p, 4 * Pn); L.opac = carve<float>(p, Pn);
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

size_t gms_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { (void)W; (void)H; return render_layout(nullptr, P).total + 512; }

int gms_render_frame(const gms_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    if (!a || !alloc || !a->workspace || !a->image || !a->invdepth || !a->radii) return set_err(GMS_E_ARG, "gms_render_frame: null argument%s%s");
    if (!a->vertices || !a->faces || !a->alpha_raw || !a->scale_raw || !a->features || !a->opacity_raw)
        return set_err(GMS_E_ARG, "gms_render_frame: model tensors required%s%s");
    const FrameModel m = {a->V, a->F, a->K, a->M, a->vertices, a->faces, a->alpha_raw, a->scale_raw, a->features, a->opacity_raw, a->eps,
                          a->segments, a->n_segments, a->alpha_activation};
    int P, rc;
    if ((rc = frame_gaussian_count("gms_render_frame", m, &P))) return rc;
    const int W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_render_workspace_bytes(P, W, H)) return set_err(GMS_E_ARG, "gms_render_frame: workspace too small%s%s");
    RenderLayout RL = render_layout(aligned_base_c(a->workspace), P);
    gms_raster_outputs out = {a->image, a->radii, a->invdepth, GMS_FORWARD_ONLY};
    std::vector<gms_expand_args> ea;
    gms_raster_inputs in;
    gms_raster_saved saved;
    if ((rc = mesh_expand_forward(m, RL.xyz, RL.scales, RL.rots, cuda_stream, &ea))) return rc;
    const FrameGaussians g = {P, a->M, RL.xyz, RL.scales, RL.rots, a->features, a->opacity_raw, RL.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

size_t gms_points_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { return gms_render_workspace_bytes(P, W, H); }

int gms_points_render_frame(const gms_points_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    if (!a || !alloc || !a->workspace || !a->image || !a->invdepth || !a->radii)
        return set_err(GMS_E_ARG, "gms_points_render_frame: null argument%s%s");
    if (!a->triangles || !a->features || !a->opacity_raw) return set_err(GMS_E_ARG, "gms_points_render_frame: model tensors required%s%s");
    if (a->P < 0) return set_err(GMS_E_ARG, "gms_points_render_frame: P < 0%s%s");
    const int P = a->P, W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_points_render_workspace_bytes(P, W, H))
        return set_err(GMS_E_ARG, "gms_points_render_frame: workspace too small%s%s");
    RenderLayout RL = render_layout(aligned_base_c(a->workspace), P);
    // pseudo-mesh triangles -> xyz = v1, (eps, exp(log s2), exp(log s3)), normalised quaternion
    gms_points_args pa;
    memset(&pa, 0, sizeof(pa));
    pa.P = P; pa.triangles = a->triangles; pa.eps = a->eps; pa.xyz = RL.xyz; pa.scaling_act = RL.scales; pa.rotation_act = RL.rots;
    int rc;
    if ((rc = gms_points_expand_forward(&pa, cuda_stream))) return rc;
    gms_raster_outputs out = {a->image, a->radii, a->invdepth, GMS_FORWARD_ONLY};
    gms_raster_inputs in;
    gms_raster_saved saved;
    const FrameGaussians g = {P, a->M, RL.xyz, RL.scales, RL.rots, a->features, a->opacity_raw, RL.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

size_t gms_pseudomesh_bind_scratch_bytes(int32_t F) {
    return align_up(16 * (size_t)(F > 0 ? F : 1)) + 256 + 512;
}

int gms_pseudomesh_bind(const gms_pseudomesh_bind_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->vertices || !a->faces || !a->n_degenerate || !a->scratch || (a->P > 0 && (!a->triangles || !a->face || !a->coeffs)))
        return set_err(GMS_E_ARG, "gms_pseudomesh_bind: null argument%s%s");
    if (a->P < 0 || a->F < 1 || a->V < 1) return set_err(GMS_E_ARG, "gms_pseudomesh_bind: need P >= 0, F >= 1, V >= 1%s%s");
    if (a->scratch_bytes < gms_pseudomesh_bind_scratch_bytes(a->F)) return set_err(GMS_E_ARG, "gms_pseudomesh_bind: scratch too small%s%s");
    char* base = reinterpret_cast<char*>(aligned_base_c(a->scratch));
    float4* cent = carve<float4>(base, a->F);
    uint32_t* n_deg = carve<uint32_t>(base, 1);
    GMS_CUDA(cudaMemsetAsync(n_deg, 0, sizeof(uint32_t), st));
    span_begin(K_MISC, st);
    k_pseudomesh_faces<<<(a->F + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, st>>>(a->F, a->vertices, a->faces, cent, n_deg);
    GMS_AFTER_LAUNCH("pseudomesh_faces", 0, st);
    span_end(st);
    uint32_t nd = 0;
    GMS_CUDA(cudaMemcpyAsync(&nd, n_deg, sizeof(nd), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaStreamSynchronize(st));
    *a->n_degenerate = (int32_t)nd;
    if ((int64_t)nd >= a->F) return set_err(GMS_E_ARG, "gms_pseudomesh_bind: every face of the mesh is degenerate%s%s");
    if (a->P == 0) return GMS_OK;
    span_begin(K_MISC, st);
    k_pseudomesh_bind<<<(a->P + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, st>>>(a->P, a->F, a->triangles, a->vertices, a->faces,
                                                                                          cent, a->face, a->coeffs);
    GMS_AFTER_LAUNCH("pseudomesh_bind", 0, st);
    span_end(st);
    return GMS_OK;
}

static bool repose_args_ok(const gms_pseudomesh_repose_args& r) {
    return r.P >= 0 && r.F >= 1 && r.V >= 1 && (r.P == 0 || (r.face && r.coeffs && r.vertices && r.faces));
}

int gms_pseudomesh_repose(const gms_pseudomesh_repose_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !repose_args_ok(*a) || (a->P > 0 && !a->triangles)) return set_err(GMS_E_ARG, "gms_pseudomesh_repose: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    span_begin(K_MISC, st);
    k_pseudomesh_repose<<<(a->P + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, st>>>(*a);
    GMS_AFTER_LAUNCH("pseudomesh_repose", 0, st);
    span_end(st);
    return GMS_OK;
}

size_t gms_bound_points_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { return gms_render_workspace_bytes(P, W, H); }

int gms_bound_points_render_frame(const gms_bound_points_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !alloc || !a->workspace || !a->image || !a->invdepth || !a->radii)
        return set_err(GMS_E_ARG, "gms_bound_points_render_frame: null argument%s%s");
    if (!a->face || !a->coeffs || !a->vertices || !a->faces || !a->features || !a->opacity_raw || !a->settings.viewmatrix)
        return set_err(GMS_E_ARG, "gms_bound_points_render_frame: model tensors required%s%s");
    if (a->P < 0 || a->F < 1 || a->V < 1) return set_err(GMS_E_ARG, "gms_bound_points_render_frame: need P >= 0, F >= 1, V >= 1%s%s");
    const int P = a->P, W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_bound_points_render_workspace_bytes(P, W, H))
        return set_err(GMS_E_ARG, "gms_bound_points_render_frame: workspace too small%s%s");
    RenderLayout RL = render_layout(aligned_base_c(a->workspace), P);
    // binding + driving pose -> re-posed triangle -> xyz = v1, (eps, exp(log s2), exp(log s3)), normalised quaternion
    if (P > 0) {
        gms_pseudomesh_repose_args r;
        memset(&r, 0, sizeof(r));
        r.P = P; r.face = a->face; r.coeffs = a->coeffs; r.V = a->V; r.F = a->F; r.vertices = a->vertices; r.faces = a->faces;
        gms_points_args pa;
        memset(&pa, 0, sizeof(pa));
        pa.P = P; pa.eps = a->eps; pa.xyz = RL.xyz; pa.scaling_act = RL.scales; pa.rotation_act = RL.rots;
        span_begin(K_EXP_FWD, st);
        k_points_bound_expand_fwd<<<(P + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, st>>>(r, pa, a->settings.viewmatrix);
        GMS_AFTER_LAUNCH("points_bound_expand_fwd", 0, st);
        span_end(st);
    }
    gms_raster_outputs out = {a->image, a->radii, a->invdepth, GMS_FORWARD_ONLY};
    gms_raster_inputs in;
    gms_raster_saved saved;
    const FrameGaussians g = {P, a->M, RL.xyz, RL.scales, RL.rots, a->features, a->opacity_raw, RL.opac};
    int rc;
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

int gms_train_frame(const gms_frame_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !alloc || !a->workspace || !a->loss || !a->gt) return set_err(GMS_E_ARG, "gms_train_frame: null argument%s%s");
    if (!a->vertices || !a->faces || !a->alpha_raw || !a->scale_raw || !a->features || !a->opacity_raw)
        return set_err(GMS_E_ARG, "gms_train_frame: model tensors required%s%s");
    if (!a->d_vertices || !a->d_alpha_raw || !a->d_scale_raw || (!a->d_features && !a->d_color_sh && !a->sh_adam) || !a->d_opacity_raw)
        return set_err(GMS_E_ARG, "gms_train_frame: gradient tensors required%s%s");
    if (a->sh_adam && (!a->sh_adam->m || !a->sh_adam->v || a->sh_adam->step < 1 || a->settings.sh_degree < 0 || a->settings.sh_degree > 3))
        return set_err(GMS_E_ARG, "gms_train_frame: bad sh_adam%s%s");
    const FrameModel m = {a->V, a->F, a->K, a->M, a->vertices, a->faces, a->alpha_raw, a->scale_raw, a->features, a->opacity_raw, a->eps,
                          a->segments, a->n_segments, a->alpha_activation};
    int P, rc;
    if ((rc = frame_gaussian_count("gms_train_frame", m, &P))) return rc;
    const int W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_frame_workspace_bytes(P, W, H)) return set_err(GMS_E_ARG, "gms_train_frame: workspace too small%s%s");
    FrameLayout FL = frame_layout(aligned_base_c(a->workspace), P, W, H);
    gms_raster_outputs out = {FL.image, FL.radii, FL.invdepth, 0};
    std::vector<gms_expand_args> ea;
    gms_raster_inputs in;
    gms_raster_saved saved;
    if ((rc = mesh_expand_forward(m, FL.xyz, FL.scales, FL.rots, cuda_stream, &ea))) return rc;
    const FrameGaussians g = {P, a->M, FL.xyz, FL.scales, FL.rots, a->features, a->opacity_raw, FL.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    // loss + dL/dimage
    gms_loss_args la;
    memset(&la, 0, sizeof(la));
    la.C = 3; la.H = H; la.W = W; la.img = FL.image; la.gt = a->gt; la.lambda_dssim = a->lambda_dssim; la.loss = a->loss;
    la.dL_dimg = FL.dimage; la.scratch = FL.loss_scratch; la.scratch_bytes = FL.loss_bytes;
    if ((rc = gms_l1_ssim_loss(&la, cuda_stream))) return rc;
    if (a->event_loss_ready) GMS_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(a->event_loss_ready), st));
    // rasterizer backward: dL/dshs goes straight to the caller's gradient buffer
    gms_raster_grads gr;
    memset(&gr, 0, sizeof(gr));
    gr.dL_dmeans3D = FL.d_xyz; gr.dL_dmeans2D = FL.d_m2d; gr.dL_dopacities = FL.d_opac;
    if (a->d_color_sh) {    // factored SH gradient: colour gradient + this camera's centre (right behind it) for gms_adam_sh_factored
        gr.dL_dcolors_sh = a->d_color_sh;
        GMS_CUDA(cudaMemcpyAsync(a->d_color_sh + 3 * (size_t)P, a->settings.campos, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    } else if (!a->sh_adam) gr.dL_dshs = a->d_features;
    gr.dL_dscales = FL.d_scales; gr.dL_drotations = FL.d_rots;
    // sh_adam: the preprocess backward updates `features` in place; it is the frame's last reader of them (the expansion
    // backward below does not read them)
    if ((rc = raster_backward_impl(&a->settings, &in, FL.radii, &saved, FL.dimage, nullptr, &gr, cuda_stream, a->d_opacity_raw, a->sh_adam)))
        return rc;
    if (a->event_sh_ready) GMS_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(a->event_sh_ready), st));
    // expansion backward (vertex gradients are accumulated with atomics: the caller keeps d_vertices zeroed)
    if ((rc = mesh_expand_backward(ea, FL.d_xyz, FL.d_scales, FL.d_rots, a->d_vertices, a->d_alpha_raw, a->d_scale_raw, cuda_stream)))
        return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

// ------------------------------------------------------------------------------------------ free Gaussians (gs, gs_flat)

static bool free_model_ok(int P, int M, int cols, const float* xyz, const float* s, const float* r, const float* f, const float* o) {
    return P >= 0 && M >= 1 && M <= 16 && (cols == 2 || cols == 3) && (P == 0 || (xyz && s && r && f && o));
}

// The activation kernels move quaternions and their gradients as float4.
static bool aligned16(const void* p) { return (reinterpret_cast<size_t>(p) & 15) == 0; }

static int free_act_fwd(int P, int cols, const float* scaling_raw, const float* rotation_raw, float eps, float* scales, float* rots,
                        cudaStream_t st) {
    if (P == 0) return GMS_OK;
    span_begin(K_EXP_FWD, st);
    k_free_act_fwd<<<(P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, st>>>(P, cols, scaling_raw, rotation_raw, eps, scales, rots);
    GMS_AFTER_LAUNCH("free_act_fwd", 0, st);
    span_end(st);
    return GMS_OK;
}

int gms_free_train_frame(const gms_free_frame_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !alloc || !a->workspace || !a->loss || !a->gt) return set_err(GMS_E_ARG, "gms_free_train_frame: null argument%s%s");
    if (!free_model_ok(a->P, a->M, a->scale_cols, a->xyz, a->scaling_raw, a->rotation_raw, a->features, a->opacity_raw))
        return set_err(GMS_E_ARG, "gms_free_train_frame: need P >= 0, 1 <= M <= 16, scale_cols 2 or 3 and every model tensor%s%s");
    const int P = a->P;
    if (P > 0 && (!a->d_xyz || !a->d_scaling_raw || !a->d_rotation_raw || (!a->d_features && !a->sh_adam) || !a->d_opacity_raw))
        return set_err(GMS_E_ARG, "gms_free_train_frame: gradient tensors required%s%s");
    if (!a->accum != !a->denom) return set_err(GMS_E_ARG, "gms_free_train_frame: accum and denom go together%s%s");
    if (!aligned16(a->rotation_raw) || !aligned16(a->d_rotation_raw))
        return set_err(GMS_E_ARG, "gms_free_train_frame: rotation_raw and d_rotation_raw must be 16-byte aligned%s%s");
    if (a->sh_adam && (!a->sh_adam->m || !a->sh_adam->v || a->sh_adam->step < 1 || a->M != 16 || a->settings.sh_degree < 0 ||
                       a->settings.sh_degree > 3))
        return set_err(GMS_E_ARG, "gms_free_train_frame: bad sh_adam%s%s");
    const int W = a->settings.image_width, H = a->settings.image_height;
    if (W <= 0 || H <= 0) return set_err(GMS_E_ARG, "gms_free_train_frame: bad image size%s%s");
    if (a->workspace_bytes < gms_frame_workspace_bytes(P, W, H)) return set_err(GMS_E_ARG, "gms_free_train_frame: workspace too small%s%s");
    FrameLayout FL = frame_layout(aligned_base_c(a->workspace), P, W, H);
    gms_raster_outputs out = {FL.image, FL.radii, FL.invdepth, 0};
    gms_raster_inputs in;
    gms_raster_saved saved;
    int rc;
    if ((rc = free_act_fwd(P, a->scale_cols, a->scaling_raw, a->rotation_raw, a->eps, FL.scales, FL.rots, st))) return rc;
    const FrameGaussians g = {P, a->M, a->xyz, FL.scales, FL.rots, a->features, a->opacity_raw, FL.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    gms_loss_args la;
    memset(&la, 0, sizeof(la));
    la.C = 3; la.H = H; la.W = W; la.img = FL.image; la.gt = a->gt; la.lambda_dssim = a->lambda_dssim; la.loss = a->loss;
    la.dL_dimg = FL.dimage; la.scratch = FL.loss_scratch; la.scratch_bytes = FL.loss_bytes;
    if ((rc = gms_l1_ssim_loss(&la, cuda_stream))) return rc;
    if (a->event_loss_ready) GMS_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(a->event_loss_ready), st));
    gms_raster_grads gr;
    memset(&gr, 0, sizeof(gr));
    gr.dL_dmeans3D = a->d_xyz; gr.dL_dmeans2D = FL.d_m2d; gr.dL_dopacities = FL.d_opac;
    if (!a->sh_adam) gr.dL_dshs = a->d_features;
    gr.dL_dscales = FL.d_scales; gr.dL_drotations = FL.d_rots;
    if ((rc = raster_backward_impl(&a->settings, &in, FL.radii, &saved, FL.dimage, nullptr, &gr, cuda_stream, a->d_opacity_raw, a->sh_adam)))
        return rc;
    if (P > 0) {
        FreeActBwd b;
        b.P = P; b.cols = a->scale_cols; b.rotation_raw = a->rotation_raw; b.scales = FL.scales;
        b.d_scales = FL.d_scales; b.d_rots = FL.d_rots; b.d_m2d = FL.d_m2d; b.radii = FL.radii;
        b.d_scaling_raw = a->d_scaling_raw; b.d_rotation_raw = a->d_rotation_raw; b.accum = a->accum; b.denom = a->denom;
        b.counters = geom_layout(aligned_base(saved.geom), P).counters;
        span_begin(K_EXP_BWD, st);
        k_free_act_bwd<<<(P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, st>>>(b);
        GMS_AFTER_LAUNCH("free_act_bwd", 0, st);
        span_end(st);
    }
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

int gms_free_render_frame(const gms_free_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !alloc || !a->workspace || !a->image || !a->invdepth || !a->radii)
        return set_err(GMS_E_ARG, "gms_free_render_frame: null argument%s%s");
    if (!free_model_ok(a->P, a->M, a->scale_cols, a->xyz, a->scaling_raw, a->rotation_raw, a->features, a->opacity_raw))
        return set_err(GMS_E_ARG, "gms_free_render_frame: need P >= 0, 1 <= M <= 16, scale_cols 2 or 3 and every model tensor%s%s");
    if (!aligned16(a->rotation_raw)) return set_err(GMS_E_ARG, "gms_free_render_frame: rotation_raw must be 16-byte aligned%s%s");
    const int P = a->P, W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_render_workspace_bytes(P, W, H)) return set_err(GMS_E_ARG, "gms_free_render_frame: workspace too small%s%s");
    RenderLayout RL = render_layout(aligned_base_c(a->workspace), P);
    int rc;
    if ((rc = free_act_fwd(P, a->scale_cols, a->scaling_raw, a->rotation_raw, a->eps, RL.scales, RL.rots, st))) return rc;
    gms_raster_outputs out = {a->image, a->radii, a->invdepth, GMS_FORWARD_ONLY};
    gms_raster_inputs in;
    gms_raster_saved saved;
    const FrameGaussians g = {P, a->M, a->xyz, RL.scales, RL.rots, a->features, a->opacity_raw, RL.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

// ------------------------------------------------------------------------------------------ gs_flame checkpoint render

// xyz from the checkpoint's activated weights and the driving pose (the product of the expansion forward, same operation
// order), scales and rotations from the checkpoint's rows as k_free_act_fwd activates them.
__global__ void __launch_bounds__(GMS_FREE_BLOCK) k_flame_act(int P, int K, const float* __restrict__ alpha, const int64_t* __restrict__ faces,
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

size_t gms_flame_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { return gms_render_workspace_bytes(P, W, H); }

int gms_flame_render_frame(const gms_flame_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !alloc || !a->workspace || !a->image || !a->invdepth || !a->radii)
        return set_err(GMS_E_ARG, "gms_flame_render_frame: null argument%s%s");
    if (!a->vertices || !a->faces || !a->alpha || !a->scaling_log || !a->rotation_raw || !a->features || !a->opacity_raw)
        return set_err(GMS_E_ARG, "gms_flame_render_frame: model tensors required%s%s");
    if (a->F < 0 || a->K < 1 || a->V < 1 || a->M < 1 || a->M > 16 || (int64_t)a->F * a->K > INT32_MAX)
        return set_err(GMS_E_ARG, "gms_flame_render_frame: need F >= 0, K >= 1, V >= 1, 1 <= M <= 16 and F*K < 2^31%s%s");
    if (!aligned16(a->rotation_raw)) return set_err(GMS_E_ARG, "gms_flame_render_frame: rotation_raw must be 16-byte aligned%s%s");
    const int P = a->F * a->K, W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_flame_render_workspace_bytes(P, W, H))
        return set_err(GMS_E_ARG, "gms_flame_render_frame: workspace too small%s%s");
    RenderLayout RL = render_layout(aligned_base_c(a->workspace), P);
    if (P > 0) {
        span_begin(K_EXP_FWD, st);
        k_flame_act<<<(P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, st>>>(P, a->K, a->alpha, a->faces, a->vertices,
                                                                                       a->scaling_log, a->rotation_raw, RL.xyz, RL.scales, RL.rots);
        GMS_AFTER_LAUNCH("flame_act", 0, st);
        span_end(st);
    }
    gms_raster_outputs out = {a->image, a->radii, a->invdepth, GMS_FORWARD_ONLY};
    gms_raster_inputs in;
    gms_raster_saved saved;
    const FrameGaussians g = {P, a->M, RL.xyz, RL.scales, RL.rots, a->features, a->opacity_raw, RL.opac};
    int rc;
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

struct DensifyScratch { int4* flags; int4* incl; void* cub; size_t cub_bytes; size_t total; };

static DensifyScratch densify_scratch(void* base, int P) {
    DensifyScratch S;
    char* p = reinterpret_cast<char*>(base);
    const int Pn = P > 0 ? P : 1;
    S.flags = carve<int4>(p, Pn); S.incl = carve<int4>(p, Pn);
    S.cub_bytes = 0;
    cub::DeviceScan::InclusiveScan(nullptr, S.cub_bytes, S.flags, S.incl, Int4Sum(), Pn);
    S.cub = p;
    p += align_up(S.cub_bytes);
    S.total = (size_t)(p - reinterpret_cast<char*>(base));
    return S;
}

size_t gms_densify_scratch_bytes(int32_t P) { return densify_scratch(nullptr, P).total + 512; }

int gms_densify_plan(const gms_densify_plan_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->result || a->P < 0 || (a->scale_cols != 2 && a->scale_cols != 3))
        return set_err(GMS_E_ARG, "gms_densify_plan: need result, P >= 0 and scale_cols 2 or 3%s%s");
    if (a->P > 0 && (!a->accum || !a->denom || !a->scaling_raw || !a->opacity_raw || !a->scratch))
        return set_err(GMS_E_ARG, "gms_densify_plan: null argument%s%s");
    if (a->P > 0 && a->scratch_bytes < gms_densify_scratch_bytes(a->P)) return set_err(GMS_E_ARG, "gms_densify_plan: scratch too small%s%s");
    memset(a->result, 0, 5 * sizeof(int32_t));
    if (a->P == 0) return GMS_OK;
    const int P = a->P;
    DensifyScratch S = densify_scratch(aligned_base_c(a->scratch), P);
    DensifyPlanK k;
    k.P = P; k.cols = a->scale_cols; k.accum = a->accum; k.denom = a->denom; k.scaling_raw = a->scaling_raw; k.opacity_raw = a->opacity_raw;
    k.eps = a->eps; k.grad_threshold = a->grad_threshold; k.split_scale = a->split_scale; k.min_opacity = a->min_opacity;
    k.max_world_scale = a->max_world_scale; k.flags = S.flags; k.fate = a->fate;
    span_begin(K_MISC, st);
    k_densify_plan<<<(P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, st>>>(k);
    GMS_AFTER_LAUNCH("densify_plan", 0, st);
    size_t tb = S.cub_bytes;
    GMS_CUDA(cub::DeviceScan::InclusiveScan(S.cub, tb, S.flags, S.incl, Int4Sum(), P, st));
    span_end(st);
    int4 tot;
    GMS_CUDA(cudaMemcpyAsync(&tot, S.incl + (P - 1), sizeof(int4), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaStreamSynchronize(st));
    const int64_t newP = (int64_t)tot.x + tot.y + 2 * (int64_t)tot.z;
    if (newP > INT32_MAX) return set_err(GMS_E_ARG, "gms_densify_plan: the densified set exceeds int32 rows%s%s");
    a->result[0] = (int32_t)newP; a->result[1] = tot.x; a->result[2] = tot.y; a->result[3] = tot.z; a->result[4] = tot.w;
    return GMS_OK;
}

static bool free_set_ok(const gms_free_set& s) { return s.xyz && s.scaling && s.rotation && s.opacity && s.features; }

int gms_densify_apply(const gms_densify_apply_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->result || a->P < 0 || a->M < 1 || a->M > 16 || (a->scale_cols != 2 && a->scale_cols != 3))
        return set_err(GMS_E_ARG, "gms_densify_apply: need result, P >= 0, 1 <= M <= 16 and scale_cols 2 or 3%s%s");
    const int32_t* r = a->result;
    if (a->new_P != r[0] || r[0] != r[1] + r[2] + 2 * r[3]) return set_err(GMS_E_ARG, "gms_densify_apply: new_P is not the plan's%s%s");
    if (a->P == 0) return GMS_OK;
    if (!a->scratch || a->scratch_bytes < gms_densify_scratch_bytes(a->P) || !a->normals)
        return set_err(GMS_E_ARG, "gms_densify_apply: scratch and normals required%s%s");
    for (int t = 0; t < 3; t++)
        if (!free_set_ok(a->src[t]) || (a->new_P > 0 && !free_set_ok(a->dst[t])))
            return set_err(GMS_E_ARG, "gms_densify_apply: every source and destination tensor is required%s%s");
    if (a->new_P == 0) return GMS_OK;
    DensifyScratch S = densify_scratch(const_cast<void*>(aligned_base_c(const_cast<void*>(a->scratch))), a->P);
    DensifyApplyK k;
    k.P = a->P; k.cols = a->scale_cols; k.F = 3 * a->M; k.eps = a->eps; k.incl = S.incl;
    k.kept = r[1]; k.clones = r[2]; k.splits = r[3]; k.normals = a->normals;
    for (int t = 0; t < 3; t++) {
        const gms_free_set& s = a->src[t];
        const gms_free_set& d = a->dst[t];
        k.src[t] = {s.xyz, s.scaling, s.rotation, s.opacity, s.features};
        k.dst[t] = {d.xyz, d.scaling, d.rotation, d.opacity, d.features};
    }
    span_begin(K_MISC, st);
    k_densify_apply<<<(a->P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, st>>>(k);
    GMS_AFTER_LAUNCH("densify_apply", 0, st);
    span_end(st);
    return GMS_OK;
}

// ---- three-nearest-neighbour mean squared distance (gms_knn.cuh)

struct KnnLayout {
    KnnBounds* part;                    // [GMS_KNN_BOUNDS_BLOCKS] partial bounding boxes
    KnnBounds* bounds;                  // [1] bounding box of the cloud
    uint32_t* code; uint32_t* code_s;   // [P] Morton codes, unsorted / sorted
    uint32_t* idx; uint32_t* idx_s;     // [P] point indices, unsorted / sorted
    float4* sorted;                     // [P] points in Morton order, w = original index
    float4* blo; float4* bhi;           // [boxes] per-box bounds
    void* cub; size_t cub_bytes; size_t total;
};

static KnnLayout knn_layout(void* base, int P) {
    KnnLayout L;
    char* p = reinterpret_cast<char*>(base);
    const int Pn = P > 0 ? P : 1, nbox = (Pn + GMS_KNN_BOX - 1) / GMS_KNN_BOX;
    L.part = carve<KnnBounds>(p, GMS_KNN_BOUNDS_BLOCKS);
    L.bounds = carve<KnnBounds>(p, 1);
    L.code = carve<uint32_t>(p, Pn); L.code_s = carve<uint32_t>(p, Pn);
    L.idx = carve<uint32_t>(p, Pn); L.idx_s = carve<uint32_t>(p, Pn);
    L.sorted = carve<float4>(p, Pn);
    L.blo = carve<float4>(p, nbox); L.bhi = carve<float4>(p, nbox);
    L.cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, L.cub_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    Pn, 0, 30);
    L.cub = p;
    p += align_up(L.cub_bytes);
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

size_t gms_knn_scratch_bytes(int32_t P) { return knn_layout(nullptr, P).total + 512; }

int gms_knn_dist2(const gms_knn_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->P < 0 || (a->P >= 1 && a->P <= 3) || a->P > INT32_MAX - GMS_KNN_BOX)
        return set_err(GMS_E_ARG, "gms_knn_dist2: need P == 0 or 4 <= P <= INT32_MAX - GMS_KNN_BOX (three other points)%s%s");
    if (a->P == 0) return GMS_OK;
    if (!a->points || !a->dist2 || !a->scratch) return set_err(GMS_E_ARG, "gms_knn_dist2: null argument%s%s");
    if (a->scratch_bytes < gms_knn_scratch_bytes(a->P)) return set_err(GMS_E_ARG, "gms_knn_dist2: scratch too small%s%s");
    const int P = a->P, nbox = (P + GMS_KNN_BOX - 1) / GMS_KNN_BOX;
    KnnLayout L = knn_layout(aligned_base_c(a->scratch), P);
    span_begin(K_MISC, st);
    k_knn_bounds<<<GMS_KNN_BOUNDS_BLOCKS, 256, 0, st>>>(P, a->points, L.part);
    GMS_AFTER_LAUNCH("knn_bounds", 0, st);
    k_knn_bounds_fold<<<1, 256, 0, st>>>(L.part, L.bounds);
    GMS_AFTER_LAUNCH("knn_bounds_fold", 0, st);
    k_knn_morton<<<(P + 255) / 256, 256, 0, st>>>(P, a->points, L.bounds, L.code, L.idx);
    GMS_AFTER_LAUNCH("knn_morton", 0, st);
    size_t tb = L.cub_bytes;
    GMS_CUDA(cub::DeviceRadixSort::SortPairs(L.cub, tb, L.code, L.code_s, L.idx, L.idx_s, P, 0, 30, st));
    k_knn_gather<<<(P + 255) / 256, 256, 0, st>>>(P, a->points, L.idx_s, L.sorted);
    GMS_AFTER_LAUNCH("knn_gather", 0, st);
    k_knn_box_bounds<<<(nbox + 7) / 8, 256, 0, st>>>(P, nbox, L.sorted, L.blo, L.bhi);
    GMS_AFTER_LAUNCH("knn_box_bounds", 0, st);
    k_knn_search<<<nbox, GMS_KNN_BOX, 0, st>>>(P, nbox, L.sorted, L.blo, L.bhi, a->dist2);
    GMS_AFTER_LAUNCH("knn_search", 0, st);
    span_end(st);
    return GMS_OK;
}

}  // extern "C"
