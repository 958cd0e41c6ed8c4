// gms_kernels.cu -- host state, workspace layouts and the C ABI of libgms_b200.so (see include/gms_b200.h for what each
// entry point replaces); the kernels live in the topic headers (gms_*.cuh).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 --shared -Xcompiler -fPIC
// No torch headers; PyTorch only provides memory and the stream on the Python side.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <stdio.h>
#include <string.h>
#include <initializer_list>
#include <utility>
#include <vector>

#include "../../include/gms_b200.h"
#define GMS_BRANCHFREE_DIV 1        // the product: branch-free correctly-rounded division / sqrt where operands are provably normal (gms_common.cuh)
#include "gms_common.cuh"
#include "gms_preprocess.cuh"
#include "gms_adam.cuh"
#include "gms_raster.cuh"
#include "gms_expand.cuh"
#include "gms_composite_fwd.cuh"
#include "gms_composite_bwd.cuh"
#include "gms_loss.cuh"
#include "gms_sort.cuh"
#include "gms_binning.cuh"
#include "gms_image.cuh"
#include "gms_free.cuh"
#include "gms_knn.cuh"
#include "gms_flame.cuh"
#include "gms_lpips.cuh"
#include "gms_alpha.cuh"
#include "gms_anomaly.cuh"

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
       K_METRICS, K_METRICS_FIN, K_LPIPS_CONV, K_LPIPS_POOL, K_LPIPS_HEAD, K_NAN_SCAN, K_COUNT };
static const char* const g_kernel_names[K_COUNT] = {"preprocess_fwd", "cub_sort_depth", "cub_scan_tiles", "emit_dups", "cub_sort_tiles",
                                                    "tile_ranges", "composite_fwd", "composite_bwd", "preprocess_bwd", "expand_fwd",
                                                    "expand_bwd", "ssim_stats", "ssim_grad", "adam", "misc",
                                                    "image_metrics", "metrics_finalize", "lpips_conv", "lpips_pool",
                                                    "lpips_head", "nan_scan"};
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

// Every kernel launch of the library: timed as `span` (K_*; -1 inside a span the caller has opened), counted, checked, and
// with `dbg` waited for, so that a fault is reported as the kernel that raised it.
template <typename... KArgs, typename... Args>
static int launch(const char* name, int span, int dbg, cudaStream_t st, dim3 grid, dim3 block, size_t smem, void (*k)(KArgs...),
                  Args&&... args) {
    if (span >= 0) span_begin(span, st);
    k<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
    GMS_AFTER_LAUNCH(name, dbg, st);
    if (span >= 0) span_end(st);
    return GMS_OK;
}

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

static inline void* aligned_base(void* p) { return reinterpret_cast<void*>(align_up(reinterpret_cast<size_t>(p))); }

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

extern "C" int gms_loss_scratch_bytes(int32_t C, int32_t H, int32_t W, size_t* bytes);

// One NaN scan of a stage's buffers into `record` (k_nan_scan): gms_nan_scan after its checks, and the training frames'
// anomaly hooks.  Empty buffers are dropped; nothing is launched when every buffer is empty.  Each buffer gets as many blocks
// as its float4 body needs at GMS_NAN_UNROLL loads per thread, at most 8 per SM (a full SM of 256-thread blocks).
static int nan_scan_launch(int stage, const gms_nan_buffer* bufs, int nb, uint64_t* record, int dbg, cudaStream_t st) {
    GmsNanTable t;
    int m = 0;
    int64_t most = 0;
    for (int i = 0; i < nb; i++) {
        if (bufs[i].n <= 0) continue;
        const int64_t to16 = (int64_t)(((16 - (reinterpret_cast<size_t>(bufs[i].ptr) & 15)) & 15) >> 2);
        GmsNanBuf& b = t.b[m++];
        b.ptr = bufs[i].ptr; b.n = bufs[i].n; b.head = to16 < b.n ? to16 : b.n;
        b.key = (uint64_t)stage << 56 | (uint64_t)bufs[i].tensor << 48;
        const int64_t n4 = (b.n - b.head) >> 2;
        most = n4 > most ? n4 : most;
    }
    if (m == 0) return GMS_OK;
    const int64_t per_block = (int64_t)GMS_NAN_BLOCK * GMS_NAN_UNROLL, cap = 8 * (int64_t)sm_count();
    int64_t gx = (most + per_block - 1) / per_block;
    gx = gx < 1 ? 1 : gx > cap ? cap : gx;
    return launch("nan_scan", K_NAN_SCAN, dbg, st, dim3((unsigned)gx, (unsigned)m), GMS_NAN_BLOCK, 0, k_nan_scan, t, record);
}

// A training frame's anomaly hook: scans the stage's buffers when the caller passed a record and selected the stage.
static int anomaly_hook(uint64_t* record, uint32_t stages, int stage, std::initializer_list<gms_nan_buffer> bufs, int dbg,
                        cudaStream_t st) {
    if (!record || !((stages >> stage) & 1u)) return GMS_OK;
    return nan_scan_launch(stage, bufs.begin(), (int)bufs.size(), record, dbg, st);
}

// ------------------------------------------------------------------------------------------ whole-frame orchestration

// The workspace of a forward-only frame: the activated Gaussians an expansion step writes, and sigmoid(opacity).
struct RenderLayout { float* xyz; float* scales; float* rots; float* opac; size_t total; };

static RenderLayout render_layout(void* base, int P) {
    RenderLayout L;
    char* p = reinterpret_cast<char*>(base);
    const size_t Pn = (size_t)(P > 0 ? P : 1);
    L.xyz = carve<float>(p, 3 * Pn); L.scales = carve<float>(p, 3 * Pn); L.rots = carve<float>(p, 4 * Pn); L.opac = carve<float>(p, Pn);
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

// The workspace of a training frame: a forward-only frame's, then the frame's own outputs, gradients and loss scratch.
struct FrameLayout {
    RenderLayout g; int32_t* radii; float* image; float* invdepth; float* dimage;
    float* d_xyz; float* d_m2d; float* d_opac; float* d_scales; float* d_rots; float* loss_scratch; size_t loss_bytes; size_t total;
};

static FrameLayout frame_layout(void* base, int P, int W, int H) {
    FrameLayout L;
    L.g = render_layout(base, P);
    char* p = reinterpret_cast<char*>(base) + L.g.total;
    const size_t Pn = (size_t)(P > 0 ? P : 1), HW = (size_t)W * H;
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
    char* base = reinterpret_cast<char*>(aligned_base(a->scratch));
    float* acc = reinterpret_cast<float*>(base);
    float* dmap = reinterpret_cast<float*>(base + 256);
    const GmsGaussWin win = ssim_window();
    GMS_CUDA(cudaMemsetAsync(acc, 0, 2 * sizeof(float), st));
    dim3 grid((W + GMS_SSIM_T - 1) / GMS_SSIM_T, (H + GMS_SSIM_T - 1) / GMS_SSIM_T, C);
    int rc;
    if ((rc = launch("ssim_stats", K_LOSS_STATS, 0, st, grid, 256, 0, k_ssim_stats, C, H, W, a->img, a->gt, win,
                     a->dL_dimg ? dmap : nullptr, acc))) return rc;
    const float inv_n = 1.0f / ((float)C * (float)H * (float)W);
    if ((rc = launch("loss_finalize", -1, 0, st, 1, 1, 0, k_loss_finalize, acc, inv_n, a->lambda_dssim, a->loss))) return rc;
    if (!a->dL_dimg) return GMS_OK;
    return launch("ssim_grad", K_LOSS_GRAD, 0, st, grid, 256, 0, k_ssim_grad, C, H, W, a->img, a->gt, win, dmap,
                  -a->lambda_dssim * inv_n, (1.f - a->lambda_dssim) * inv_n, a->dL_dloss, a->dL_dimg);
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
    float* part = reinterpret_cast<float*>(aligned_base(a->scratch));
    const GmsGaussWin win = ssim_window();
    dim3 grid((W + GMS_SSIM_T - 1) / GMS_SSIM_T, (H + GMS_SSIM_T - 1) / GMS_SSIM_T, C);
    if ((rc = launch("image_metrics", K_METRICS, 0, st, grid, 256, 0, a->quantize ? k_image_metrics<1> : k_image_metrics<0>, C, H, W,
                     a->img, a->gt, win, part))) return rc;
    return launch("metrics_finalize", K_METRICS_FIN, 0, st, 1, 256, 0, k_metrics_finalize, C, metric_tiles(H, W),
                  1.0 / ((double)H * (double)W), part, a->out);
}

// VGG16 up to relu5_3 (torchvision's vgg16().features): conv l reads Cin[l] channels and writes Cout[l]; the target maps are
// the outputs of convs 1, 3, 6, 9 and 12 (features' 1-based layers 4, 9, 16, 23, 30), each followed by a 2x2 max-pool but
// the last.
static const int kLpipsCin[13] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
static const int kLpipsCout[13] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
static const int kLpipsTarget[5] = {1, 3, 6, 9, 12};
static int lpips_kp(int l) { return l == 0 ? 32 : 9 * kLpipsCin[l]; }

struct LpipsLayout {
    float* act[2];      // ping-pong [2,H,W,64] (every later level holds at most as many floats)
    double* part[5];    // per target layer: one partial per head block
    int blocks[5];
    size_t total;
};
static LpipsLayout lpips_layout(void* base, int H, int W) {
    LpipsLayout L;
    char* p = reinterpret_cast<char*>(base);
    for (int i = 0; i < 2; i++) L.act[i] = carve<float>(p, (size_t)2 * H * W * 64);
    for (int l = 0; l < 5; l++) {
        const size_t hw = (size_t)(H >> l) * (W >> l);
        L.blocks[l] = (int)((hw + GMS_LPIPS_HEAD_PIX - 1) / GMS_LPIPS_HEAD_PIX);
        L.part[l] = carve<double>(p, L.blocks[l]);
    }
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

size_t gms_lpips_scratch_bytes(int32_t H, int32_t W) {
    if (H < 16 || W < 16) return 0;
    return lpips_layout(nullptr, H, W).total + 256;
}

int gms_lpips_vgg(const gms_lpips_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !a->img || !a->gt || !a->weights || !a->out || !a->scratch) return set_err(GMS_E_ARG, "gms_lpips_vgg: null argument%s%s");
    if (a->H < 16 || a->W < 16) return set_err(GMS_E_ARG, "gms_lpips_vgg: H and W must be at least 16%s%s");
    if (a->scratch_bytes < gms_lpips_scratch_bytes(a->H, a->W)) return set_err(GMS_E_ARG, "gms_lpips_vgg: scratch too small%s%s");
    const LpipsLayout L = lpips_layout(aligned_base(a->scratch), a->H, a->W);
    const float* w = a->weights;
    const float* lin = a->weights;
    for (int l = 0; l < 13; l++) lin += (size_t)kLpipsCout[l] * (lpips_kp(l) + 1);
    LpipsFinal fin;
    int H = a->H, W = a->W, cur = 0, target = 0, rc;
    const float* in = nullptr;
    for (int l = 0; l < 13; l++) {
        LpipsConv c;
        c.in = in; c.img = a->img; c.gt = a->gt; c.w = w; c.bias = w + (size_t)kLpipsCout[l] * lpips_kp(l);
        c.out = L.act[cur]; c.H = H; c.W = W; c.Cin = kLpipsCin[l]; c.Cout = kLpipsCout[l]; c.Kp = lpips_kp(l);
        w = c.bias + kLpipsCout[l];
        const dim3 grid((unsigned)((2 * (size_t)H * W + GMS_LPIPS_BM - 1) / GMS_LPIPS_BM), (unsigned)(c.Cout / GMS_LPIPS_BN));
        if ((rc = launch("lpips_conv", K_LPIPS_CONV, 0, st, grid, 128, 0, l == 0 ? k_lpips_conv<true> : k_lpips_conv<false>, c))) return rc;
        in = c.out;
        if (l != kLpipsTarget[target]) { cur ^= 1; continue; }
        const int C = c.Cout, hw = H * W;
        void (*head)(const float*, int, const float*, double*) =
            C == 64 ? k_lpips_head<2> : C == 128 ? k_lpips_head<4> : C == 256 ? k_lpips_head<8> : k_lpips_head<16>;
        if ((rc = launch("lpips_head", K_LPIPS_HEAD, 0, st, L.blocks[target], 256, 0, head, c.out, hw, lin, L.part[target]))) return rc;
        fin.part[target] = L.part[target]; fin.blocks[target] = L.blocks[target]; fin.inv_hw[target] = 1.0 / (double)hw;
        lin += C;
        if (++target == 5) break;
        const size_t n4 = (size_t)2 * (H / 2) * (W / 2) * (C / 4);
        if ((rc = launch("lpips_pool", K_LPIPS_POOL, 0, st, (unsigned)((n4 + 255) / 256), 256, 0, k_lpips_pool, c.out, H, W, C,
                         L.act[cur ^ 1]))) return rc;
        in = L.act[cur ^ 1];
        H /= 2; W /= 2;
    }
    return launch("lpips_finalize", -1, 0, st, 1, 256, 0, k_lpips_finalize, fin, a->out);
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
    return launch("adam", K_ADAM, 0, st, (unsigned)((nthreads + 255) / 256), 256, 0, k_adam, k);
}

int gms_image_quantize(const float* chw, uint8_t* out, int32_t C, int32_t H, int32_t W, int32_t row_prefix, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!chw || !out || C <= 0 || C > 4 || H <= 0 || W <= 0 || row_prefix < 0 || row_prefix > 16) return set_err(GMS_E_ARG, "gms_image_quantize: bad arguments%s%s");
    return launch("image_quantize", -1, 0, st, dim3((W + 255) / 256, H), 256, 0, k_image_quantize, chw, out, C, H, W, row_prefix);
}

int gms_image_clamp_u8(const float* chw, uint8_t* hwc, int32_t C, int32_t H, int32_t W, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!chw || !hwc || C <= 0 || C > 4 || H <= 0 || H > 65535 || W <= 0) return set_err(GMS_E_ARG, "gms_image_clamp_u8: bad arguments%s%s");
    return launch("image_clamp_u8", -1, 0, st, dim3((W + 255) / 256, H), 256, 0, k_image_clamp_u8, chw, hwc, C, H, W);
}

int gms_image_dequantize(const uint8_t* src, int32_t src_is_hwc, float* chw, int32_t C, int32_t H, int32_t W, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!src || !chw || C <= 0 || C > 4 || H <= 0 || W <= 0) return set_err(GMS_E_ARG, "gms_image_dequantize: bad arguments%s%s");
    return launch("image_dequantize", -1, 0, st, dim3((W + 255) / 256, H), 256, 0, k_image_dequantize, src, src_is_hwc, chw, C, H, W);
}

int gms_image_composite_rgba(const uint8_t* rgba, uint8_t* rgb, int32_t H, int32_t W, int32_t white_background, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!rgba || !rgb || H <= 0 || W <= 0 || (white_background != 0 && white_background != 1) ||
        reinterpret_cast<size_t>(rgba) % 4 != 0)
        return set_err(GMS_E_ARG, "gms_image_composite_rgba: bad arguments%s%s");
    const long long npix = (long long)H * W;
    return launch("image_composite_rgba", -1, 0, st, (unsigned)((npix + 255) / 256), 256, 0, k_image_composite_rgba,
                  reinterpret_cast<const uchar4*>(rgba), rgb, npix, white_background ? 1.0 : 0.0);
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
        const int rc = launch("resize_h_u8", -1, 0, st, dim3((a->out_w + 255) / 256, rows), 256, 0, k_resize_h_u8, a->src, a->in_w, out,
                              a->out_w, row0, a->bounds_h, a->coeffs_h, a->ksize_h);
        if (rc) return rc;
    }
    if (!vert) return GMS_OK;
    const uint8_t* in = horiz ? a->scratch : a->src;
    const int row0 = horiz ? a->row0 : 0;
    return launch("resize_v_u8", -1, 0, st, dim3((a->out_w + 255) / 256, a->out_h), 256, 0, k_resize_v_u8, in, a->out_w, a->dst, row0,
                  a->bounds_v, a->coeffs_v, a->ksize_v);
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
    return launch("adam_sh", K_ADAM, 0, st, (a->P + 127) / 128, 128, 0, g_opt_adam_sh_ieee ? k_adam_sh<true> : k_adam_sh<false>, k);
}

int gms_frame_views(void* workspace, int32_t P, int32_t W, int32_t H, gms_frame_view* v) {
    if (!workspace || !v) return set_err(GMS_E_ARG, "gms_frame_views: null argument%s%s");
    FrameLayout FL = frame_layout(aligned_base(workspace), P, W, H);
    v->xyz = FL.g.xyz; v->scales = FL.g.scales; v->rotations = FL.g.rots; v->opacities = FL.g.opac; v->radii = FL.radii;
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

// The end of a forward with a binned point list: tiles in launch order, then the composite forward, which writes the
// per-quad survivor lists to `surv` when `emit`.
static int composite_forward(const gms_raster_settings* s, const gms_raster_outputs* out, const ImageLayout& IL, const float4* rec,
                             const uint32_t* point_list, bool emit, uint32_t* surv, int T, cudaStream_t st) {
    const int W = s->image_width, H = s->image_height, gx = (W + GMS_TILE - 1) / GMS_TILE;
    const int dbg = s->debug;
    int rc;
    if (g_opt_tile_order && (rc = launch("tile_order", -1, dbg, st, 1, 1024, 0, k_tile_order, T, IL.ranges, IL.tile_order))) return rc;
    const int* to = g_opt_tile_order ? IL.tile_order : nullptr;
    if (g_opt_fwd == 3)
        return launch("composite_fwd", K_COMP_FWD, dbg, st, T, GMS_CB, 0, k_composite_fwd3, IL.ranges, to, point_list, rec, W, H, gx, s->bg,
                      out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth);
    return launch("composite_fwd", K_COMP_FWD, dbg, st, T, GMS_CB, 0, emit ? k_composite_fwd2<true> : k_composite_fwd2<false>, IL.ranges,
                  to, point_list, rec, W, H, gx, s->bg, out->out_color, IL.final_T, IL.n_contrib, out->out_invdepth,
                  emit ? surv : nullptr, emit ? IL.nsurv : nullptr);
}

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

    const size_t HW = (size_t)W * H;
    auto fill_background = [&]() {
        return launch("fill_background", -1, dbg, st, (unsigned)((HW + 255) / 256), 256, 0, k_fill_background, W, H, s->bg, out->out_color,
                      out->out_invdepth);
    };
    if (P == 0) {   // stock: returns background-only images without launching the pipeline
        if ((rc = fill_background())) return rc;
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
    const bool staged = g_opt_sh_staged && pa.shs && pa.M == 16;
    if ((rc = launch("preprocess_fwd", K_PRE_FWD, dbg, st, (P + 127) / 128, 128, 0, staged ? k_preprocess_fwd<true> : k_preprocess_fwd<false>,
                     pa, out->radii, GL.rec, GL.cov3D, GL.clamped, GL.tiles, GL.dkey, GL.idx, GL.rect, GL.counters))) return rc;

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
        // the sort's device-side N: a launch error is caught by gms_radix_sort_pairs's check; gms_launch_count leaves it out
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
            return composite_forward(s, out, IL, GL.rec, point_list, emit, surv, T, st);
        } else {
            if ((rc = fill_background())) return rc;
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
        auto emit_dups = [&](auto k, auto* keys) {
            return launch("emit_dups", K_EMIT, dbg, st, (P + 255) / 256, 256, 0, k, P, gx, order, GL.offs, GL.rect, keys, ev, g_opt_warp_emit,
                          cap32);
        };
        if ((rc = k16 ? emit_dups(k_emit_dups<uint16_t>, reinterpret_cast<uint16_t*>(ek)) : emit_dups(k_emit_dups<uint32_t>, ek))) return rc;
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
        auto tile_ranges = [&](auto k, const auto* keys) {
            return launch("tile_ranges", K_RANGES, dbg, st, (unsigned)((cap + 255) / 256), 256, 0, k, cap, keys, IL.ranges, (uint32_t)T,
                          GL.offs + (P - 1), GL.counters, n_host);
        };
        if ((rc = k16 ? tile_ranges(k_tile_ranges<uint16_t>, reinterpret_cast<const uint16_t*>(BL.keys_out))
                      : tile_ranges(k_tile_ranges<uint32_t>, BL.keys_out))) return rc;
        return composite_forward(s, out, IL, GL.rec, BL.vals_out, emit, BL.surv, T, st);
    } else {
        if ((rc = fill_background())) return rc;
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
                                const gms_raster_grads* gr, void* cuda_stream, float* dopac_raw, const gms_sh_adam* sh_adam,
                                uint64_t* anomaly, uint32_t anomaly_stages) {
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
        const int* to = g_opt_tile_order ? IL.tile_order : nullptr;
        const bool depth = dL_dout_invdepth != nullptr;
        const bool lists = (saved->flags & 2) != 0;       // the forward wrote per-quad survivor lists
        const uint32_t* surv = !lists ? nullptr : !counting ? BL.surv :
            reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(BL.vals_out) + align_up((size_t)saved->binning_capacity * sizeof(uint32_t)));
        // [bwd_minblocks: >= 8, >= 6, 5, else 4][depth]
        decltype(&k_composite_bwd5<4, false>) const bwd5[4][2] = {{k_composite_bwd5<8, false>, k_composite_bwd5<8, true>},
            {k_composite_bwd5<6, false>, k_composite_bwd5<6, true>}, {k_composite_bwd5<5, false>, k_composite_bwd5<5, true>},
            {k_composite_bwd5<4, false>, k_composite_bwd5<4, true>}};
        decltype(&k_composite_bwd3<4, false>) const bwd3[4][2] = {{k_composite_bwd3<8, false>, k_composite_bwd3<8, true>},
            {k_composite_bwd3<6, false>, k_composite_bwd3<6, true>}, {k_composite_bwd3<5, false>, k_composite_bwd3<5, true>},
            {k_composite_bwd3<4, false>, k_composite_bwd3<4, true>}};
        const int mb = g_opt_bwd_minb >= 8 ? 0 : g_opt_bwd_minb >= 6 ? 1 : g_opt_bwd_minb == 5 ? 2 : 3;
        auto composite_bwd = [&](auto k, auto... lists_args) {
            return launch("composite_bwd", K_COMP_BWD, dbg, st, T, GMS_CB, 0, k, IL.ranges, to, BL.vals_out, GL.rec, W, H, gx, s->bg,
                          IL.final_T, IL.n_contrib, dL_dout_color, dL_dout_invdepth, GL.dgeom, lists_args...);
        };
        if ((rc = lists ? composite_bwd(bwd5[mb][depth], surv, IL.nsurv) : composite_bwd(bwd3[mb][depth]))) return rc;
    }
    if ((rc = anomaly_hook(anomaly, anomaly_stages, GMS_ANOMALY_COMPOSITE_BWD,
                           {{reinterpret_cast<const float*>(GL.dgeom), 12 * (int64_t)P, GMS_ANOMALY_DGEOM}}, dbg, st))) return rc;
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
    const bool minb4 = g_opt_pre_bwd_minb >= 4;
    void (*k)(PreBwdArgs) = k_preprocess_bwd<0, 1>;
    if (sh_adam) {          // factored SH gradient applied in place: the SH Adam step of the frame (gms_sh_adam)
        if (b.f.M != 16 || !b.f.shs) return set_err(GMS_E_ARG, "sh_adam needs shs with 16 coefficients%s%s");
        b.dshs = nullptr;
        b.sh_p = const_cast<float*>(b.f.shs); b.sh_m = sh_adam->m; b.sh_v = sh_adam->v;
        b.sh_adam = adam_sh_const(sh_adam->lr_dc, sh_adam->lr_rest, sh_adam->beta1, sh_adam->beta2, sh_adam->eps, sh_adam->step);
        if (g_opt_adam_sh_ieee) k = minb4 ? k_preprocess_bwd<1, 4, true, true, true> : k_preprocess_bwd<1, 1, true, true, true>;
        else k = minb4 ? k_preprocess_bwd<1, 4, true, true> : k_preprocess_bwd<1, 1, true, true>;
    } else if (b.dcol_sh) {        // factored SH gradient
        if (b.f.M != 16 || !b.f.shs) return set_err(GMS_E_ARG, "dL_dcolors_sh needs shs with 16 coefficients%s%s");
        b.dshs = nullptr;
        k = minb4 ? k_preprocess_bwd<1, 4, true> : k_preprocess_bwd<1, 1, true>;
    } else if (g_opt_sh_staged && b.f.shs && b.dshs && b.f.M == 16) {
        if (g_opt_sh_staged == 2) k = minb4 ? k_preprocess_bwd<2, 4> : k_preprocess_bwd<2, 1>;
        else k = minb4 ? k_preprocess_bwd<1, 4> : k_preprocess_bwd<1, 1>;
    }
    if ((rc = launch("preprocess_bwd", K_PRE_BWD, dbg, st, (P + 127) / 128, 128, 0, k, b))) return rc;
    // (a buffer the call did not write is NULL and counts 0 floats)
    const int64_t Pn = P;
    return anomaly_hook(anomaly, anomaly_stages, GMS_ANOMALY_PREPROCESS_BWD,
                        {{b.dmeans3D, 3 * Pn, GMS_ANOMALY_DMEANS3D}, {b.dscales, b.dscales ? 3 * Pn : 0, GMS_ANOMALY_DSCALES},
                         {b.drots, b.drots ? 4 * Pn : 0, GMS_ANOMALY_DROTATIONS},
                         {dopac_raw ? dopac_raw : b.dopac, Pn, GMS_ANOMALY_DOPACITY_RAW},
                         {b.dshs, b.dshs ? 3 * Pn * b.f.M : 0, GMS_ANOMALY_DSHS},
                         {b.dcol_sh, b.dcol_sh ? 3 * Pn : 0, GMS_ANOMALY_DCOLOR_SH}}, dbg, st);
}

int gms_rasterize_backward(const gms_raster_settings* s, const gms_raster_inputs* in, const int32_t* radii,
                           const gms_raster_saved* saved, const float* dL_dout_color, const float* dL_dout_invdepth,
                           const gms_raster_grads* gr, void* cuda_stream) {
    return raster_backward_impl(s, in, radii, saved, dL_dout_color, dL_dout_invdepth, gr, cuda_stream, nullptr, nullptr, nullptr, 0);
}

int gms_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present, void* cuda_stream) {
    (void)projmatrix;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (P <= 0) return GMS_OK;
    return launch("mark_visible", -1, 0, st, (P + 255) / 256, 256, 0, k_mark_visible, P, means3D, viewmatrix, present);
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
        if (saved->flags & 2)       // counting binning: the survivor lists follow the point list (raster_forward_impl)
            v->surv = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(v->point_list) +
                                                        align_up((size_t)saved->binning_capacity * sizeof(uint32_t)));
    } else if (saved->binning && saved->binning_capacity > 0) {
        BinLayout BL = bin_layout(aligned_base(saved->binning), saved->binning_capacity);
        v->point_list = BL.vals_out; v->tile_keys = (saved->flags & 4) ? nullptr : BL.keys_out;     // (16-bit keys: callers derive them from the ranges)
        if (saved->flags & 2) v->surv = BL.surv;
    }
    if (v->surv && saved->image) v->nsurv = image_layout(aligned_base(saved->image), W, H).nsurv;
    if (!v->nsurv) v->surv = nullptr;
    return GMS_OK;
}

int gms_debug_unpack(const gms_raster_saved* saved, int32_t P, const int32_t* radii, float* means2D, float* depths,
                     float* conic_opacity, float* rgb, uint8_t* clamped, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!saved || !saved->geom || P <= 0) return set_err(GMS_E_ARG, "nothing to unpack%s%s");
    GeomLayout GL = geom_layout(aligned_base(saved->geom), P);
    return launch("unpack", -1, 0, st, (P + 255) / 256, 256, 0, k_unpack, P, GL.rec, GL.clamped, GL.dkey, radii, means2D, depths,
                  conic_opacity, rgb, clamped);
}

// floats of shared memory per Gaussian row of the staged forward (host side: sizing the launch)
static int exp_fwd_stage_width(const gms_expand_args& a) {
    return 3 + 1 + (a.alpha ? 3 : 0) + (a.xyz ? 3 : 0) + (a.scaling_log ? 3 : 0) + (a.scaling_act ? 3 : 0) +
           (a.rotation_raw ? 4 : 0) + (a.rotation_act ? 4 : 0);
}

// Which expansion kernels a call runs: one warp per face for softmax weights with many splats per face, else one thread.
static bool expand_wide(const gms_expand_args& a) {
    return a.alpha_activation == GMS_ALPHA_SOFTMAX && a.K >= GMS_EXP_WIDE_MIN_K;
}

int gms_expand_forward(const gms_expand_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->F < 0 || a->K <= 0) return set_err(GMS_E_ARG, "bad expansion sizes%s%s");
    if (!a->triangles_in && (!a->vertices || !a->faces)) return set_err(GMS_E_ARG, "vertices/faces or triangles_in required%s%s");
    if (!a->alpha_raw || !a->scale_raw) return set_err(GMS_E_ARG, "_alpha and _scale required%s%s");
    if (a->alpha_activation != GMS_ALPHA_RELU && a->alpha_activation != GMS_ALPHA_SOFTMAX)
        return set_err(GMS_E_ARG, "alpha_activation must be 0 (relu) or 1 (softmax)%s%s");
    if (a->F == 0) return GMS_OK;
    if (expand_wide(*a))
        return launch("expand_fwd", K_EXP_FWD, 0, st, (a->F + GMS_EXP_WIDE_BLOCK / 32 - 1) / (GMS_EXP_WIDE_BLOCK / 32), GMS_EXP_WIDE_BLOCK, 0,
                      k_expand_wide_fwd, *a);
    const bool softmax = a->alpha_activation == GMS_ALPHA_SOFTMAX;
    const size_t smem = (size_t)GMS_EXP_BLOCK * a->K * exp_fwd_stage_width(*a) * sizeof(float);
    const bool staged = smem <= 48 * 1024;
    void (*k)(gms_expand_args) = softmax ? (staged ? k_expand_fwd<true, GMS_ALPHA_SOFTMAX> : k_expand_fwd<false, GMS_ALPHA_SOFTMAX>)
                                         : (staged ? k_expand_fwd<true, GMS_ALPHA_RELU> : k_expand_fwd<false, GMS_ALPHA_RELU>);
    return launch("expand_fwd", K_EXP_FWD, 0, st, (a->F + GMS_EXP_BLOCK - 1) / GMS_EXP_BLOCK, GMS_EXP_BLOCK, staged ? smem : 0, k, *a);
}

int gms_points_expand_forward(const gms_points_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->P < 0 || !a->triangles) return set_err(GMS_E_ARG, "gms_points_expand_forward: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    return launch("points_expand_fwd", K_EXP_FWD, 0, st, (a->P + 127) / 128, 128, 0, k_points_expand_fwd, *a);
}

int gms_points_prepare_vertices(const gms_points_vertices_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->P < 0 || (a->scaling_cols != 2 && a->scaling_cols != 3))
        return set_err(GMS_E_ARG, "gms_points_prepare_vertices: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    if (!a->xyz || !a->scaling_log || !a->rotation_raw || !a->triangles)
        return set_err(GMS_E_ARG, "gms_points_prepare_vertices: null buffer%s%s");
    return launch("points_vertices", K_EXP_FWD, 0, st, (a->P + 127) / 128, 128, 0, k_points_vertices, *a);
}

int gms_expand_backward(const gms_expand_args* a, const gms_expand_grads* g, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !g || a->F < 0 || a->K <= 0) return set_err(GMS_E_ARG, "bad expansion sizes%s%s");
    if (!a->triangles_in && (!a->vertices || !a->faces)) return set_err(GMS_E_ARG, "vertices/faces or triangles_in required%s%s");
    if (!a->alpha_raw || !a->scale_raw) return set_err(GMS_E_ARG, "_alpha and _scale required%s%s");
    if (a->alpha_activation != GMS_ALPHA_RELU && a->alpha_activation != GMS_ALPHA_SOFTMAX)
        return set_err(GMS_E_ARG, "alpha_activation must be 0 (relu) or 1 (softmax)%s%s");
    if (a->F == 0) return GMS_OK;
    if (expand_wide(*a))
        return launch("expand_bwd", K_EXP_BWD, 0, st, (a->F + GMS_EXP_WIDE_BLOCK / 32 - 1) / (GMS_EXP_WIDE_BLOCK / 32), GMS_EXP_WIDE_BLOCK, 0,
                      k_expand_wide_bwd, *a, *g);
    return launch("expand_bwd", K_EXP_BWD, 0, st, (a->F + GMS_EXP_BLOCK - 1) / GMS_EXP_BLOCK, GMS_EXP_BLOCK, 0,
                  a->alpha_activation == GMS_ALPHA_SOFTMAX ? k_expand_bwd<GMS_ALPHA_SOFTMAX> : k_expand_bwd<GMS_ALPHA_RELU>, *a, *g);
}

size_t gms_frame_workspace_bytes(int32_t P, int32_t W, int32_t H) { return frame_layout(nullptr, P, W, H).total + 512; }

// A whole frame's forward is the model's own expansion step followed by one rasterizer forward, frame_raster_forward, which
// every one-call frame shares.  The expansion writes activated Gaussians (xyz, scales, unit quaternions) into the frame's
// workspace.
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

size_t gms_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { (void)W; (void)H; return render_layout(nullptr, P).total + 512; }

// The active SH degree against the model's coefficient rows, checked by every frame with its model, before its first launch
// (raster_forward_impl repeats it for the plain rasterizer ABI, after a frame's expansion step has already run).
static int frame_sh_check(const char* fn, int sh_degree, int M) {
    if (sh_degree < 0 || sh_degree > 3) return set_err(GMS_E_ARG, "%s: sh_degree must be 0..3%s", fn);
    if ((sh_degree + 1) * (sh_degree + 1) > M) return set_err(GMS_E_ARG, "%s: sh_degree needs more coefficients than M%s", fn);
    return GMS_OK;
}

extern "C++" {      // templates need C++ linkage

// A forward-only frame around the model's own checks and expansion step: the output checks; check_model(&P), which checks
// the model and gives its Gaussian count; the SH degree check; the workspace check; expand(P, RL, &xyz) into the render layout (free Gaussians
// point xyz at the model's own centres); one rasterizer forward; num_rendered.  Every gms_*_render_args names its
// settings, output, workspace and capacity fields alike.
template <typename Args, typename CheckModel, typename Expand>
static int render_frame(const char* fn, const Args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream, CheckModel check_model,
                        Expand expand) {
    if (!a || !alloc || !a->workspace || !a->image || !a->invdepth || !a->radii) return set_err(GMS_E_ARG, "%s: null argument%s", fn);
    int P, rc;
    if ((rc = check_model(&P))) return rc;
    if ((rc = frame_sh_check(fn, a->settings.sh_degree, a->M))) return rc;
    if (a->workspace_bytes < gms_render_workspace_bytes(P, a->settings.image_width, a->settings.image_height))
        return set_err(GMS_E_ARG, "%s: workspace too small%s", fn);
    const RenderLayout RL = render_layout(aligned_base(a->workspace), P);
    const float* xyz = RL.xyz;
    if ((rc = expand(P, RL, &xyz))) return rc;
    gms_raster_outputs out = {a->image, a->radii, a->invdepth, GMS_FORWARD_ONLY};
    gms_raster_inputs in;
    gms_raster_saved saved;
    const FrameGaussians g = {P, a->M, xyz, RL.scales, RL.rots, a->features, a->opacity_raw, RL.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

// What both training frames do after their forward: the L1+SSIM loss and dL/dimage, event_loss_ready, then the rasterizer
// backward into the workspace's gradients, dL/dmeans3D into d_xyz.  dL/dshs goes to d_features; with d_color_sh, the
// factored colour gradient goes there instead, with this camera's centre right behind it (for gms_adam_sh_factored); with
// sh_adam, neither: the preprocess backward updates `features` in place.
template <typename Args>
static int frame_loss_backward(const Args* a, const FrameLayout& FL, const gms_raster_inputs& in, const gms_raster_saved& saved,
                               float* d_xyz, float* d_color_sh, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    gms_loss_args la;
    memset(&la, 0, sizeof(la));
    la.C = 3; la.H = a->settings.image_height; la.W = a->settings.image_width; la.img = FL.image; la.gt = a->gt;
    la.lambda_dssim = a->lambda_dssim; la.loss = a->loss;
    la.dL_dimg = FL.dimage; la.scratch = FL.loss_scratch; la.scratch_bytes = FL.loss_bytes;
    int rc;
    if ((rc = gms_l1_ssim_loss(&la, cuda_stream))) return rc;
    if (a->event_loss_ready) GMS_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(a->event_loss_ready), st));
    if ((rc = anomaly_hook(a->anomaly, a->anomaly_stages, GMS_ANOMALY_LOSS, {{FL.dimage, 3 * (int64_t)la.H * la.W, GMS_ANOMALY_DIMAGE}}, 0,
                           st))) return rc;
    gms_raster_grads gr;
    memset(&gr, 0, sizeof(gr));
    gr.dL_dmeans3D = d_xyz; gr.dL_dmeans2D = FL.d_m2d; gr.dL_dopacities = FL.d_opac;
    if (d_color_sh) {
        gr.dL_dcolors_sh = d_color_sh;
        GMS_CUDA(cudaMemcpyAsync(d_color_sh + 3 * (size_t)in.P, a->settings.campos, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    } else if (!a->sh_adam) gr.dL_dshs = a->d_features;
    gr.dL_dscales = FL.d_scales; gr.dL_drotations = FL.d_rots;
    return raster_backward_impl(&a->settings, &in, FL.radii, &saved, FL.dimage, nullptr, &gr, cuda_stream, a->d_opacity_raw, a->sh_adam,
                                a->anomaly, a->anomaly_stages);
}

}   // extern "C++"

int gms_render_frame(const gms_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    FrameModel m;
    std::vector<gms_expand_args> ea;
    return render_frame("gms_render_frame", a, alloc, alloc_user, cuda_stream,
        [&](int* P) {
            if (!a->vertices || !a->faces || !a->alpha_raw || !a->scale_raw || !a->features || !a->opacity_raw)
                return set_err(GMS_E_ARG, "gms_render_frame: model tensors required%s%s");
            m = {a->V, a->F, a->K, a->M, a->vertices, a->faces, a->alpha_raw, a->scale_raw, a->features, a->opacity_raw, a->eps,
                 a->segments, a->n_segments, a->alpha_activation};
            return frame_gaussian_count("gms_render_frame", m, P);
        },
        [&](int, const RenderLayout& RL, const float**) { return mesh_expand_forward(m, RL.xyz, RL.scales, RL.rots, cuda_stream, &ea); });
}

size_t gms_points_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { return gms_render_workspace_bytes(P, W, H); }

int gms_points_render_frame(const gms_points_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    return render_frame("gms_points_render_frame", a, alloc, alloc_user, cuda_stream,
        [&](int* P) {
            if (!a->triangles || !a->features || !a->opacity_raw) return set_err(GMS_E_ARG, "gms_points_render_frame: model tensors required%s%s");
            if (a->P < 0) return set_err(GMS_E_ARG, "gms_points_render_frame: P < 0%s%s");
            *P = a->P;
            return GMS_OK;
        },
        [&](int P, const RenderLayout& RL, const float**) {
            // pseudo-mesh triangles -> xyz = v1, (eps, exp(log s2), exp(log s3)), normalised quaternion
            gms_points_args pa;
            memset(&pa, 0, sizeof(pa));
            pa.P = P; pa.triangles = a->triangles; pa.eps = a->eps; pa.xyz = RL.xyz; pa.scaling_act = RL.scales; pa.rotation_act = RL.rots;
            return gms_points_expand_forward(&pa, cuda_stream);
        });
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
    char* base = reinterpret_cast<char*>(aligned_base(a->scratch));
    float4* cent = carve<float4>(base, a->F);
    uint32_t* n_deg = carve<uint32_t>(base, 1);
    GMS_CUDA(cudaMemsetAsync(n_deg, 0, sizeof(uint32_t), st));
    int rc;
    if ((rc = launch("pseudomesh_faces", K_MISC, 0, st, (a->F + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, k_pseudomesh_faces, a->F,
                     a->vertices, a->faces, cent, n_deg))) return rc;
    uint32_t nd = 0;
    GMS_CUDA(cudaMemcpyAsync(&nd, n_deg, sizeof(nd), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaStreamSynchronize(st));
    *a->n_degenerate = (int32_t)nd;
    if ((int64_t)nd >= a->F) return set_err(GMS_E_ARG, "gms_pseudomesh_bind: every face of the mesh is degenerate%s%s");
    if (a->P == 0) return GMS_OK;
    return launch("pseudomesh_bind", K_MISC, 0, st, (a->P + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, k_pseudomesh_bind, a->P, a->F,
                  a->triangles, a->vertices, a->faces, cent, a->face, a->coeffs);
}

static bool repose_args_ok(const gms_pseudomesh_repose_args& r) {
    return r.P >= 0 && r.F >= 1 && r.V >= 1 && (r.P == 0 || (r.face && r.coeffs && r.vertices && r.faces));
}

int gms_pseudomesh_repose(const gms_pseudomesh_repose_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !repose_args_ok(*a) || (a->P > 0 && !a->triangles)) return set_err(GMS_E_ARG, "gms_pseudomesh_repose: bad arguments%s%s");
    if (a->P == 0) return GMS_OK;
    return launch("pseudomesh_repose", K_MISC, 0, st, (a->P + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0, k_pseudomesh_repose, *a);
}

size_t gms_bound_points_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { return gms_render_workspace_bytes(P, W, H); }

int gms_bound_points_render_frame(const gms_bound_points_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    return render_frame("gms_bound_points_render_frame", a, alloc, alloc_user, cuda_stream,
        [&](int* P) {
            if (!a->face || !a->coeffs || !a->vertices || !a->faces || !a->features || !a->opacity_raw || !a->settings.viewmatrix)
                return set_err(GMS_E_ARG, "gms_bound_points_render_frame: model tensors required%s%s");
            if (a->P < 0 || a->F < 1 || a->V < 1) return set_err(GMS_E_ARG, "gms_bound_points_render_frame: need P >= 0, F >= 1, V >= 1%s%s");
            *P = a->P;
            return GMS_OK;
        },
        [&](int P, const RenderLayout& RL, const float**) {
            // binding + driving pose -> re-posed triangle -> xyz = v1, (eps, exp(log s2), exp(log s3)), normalised quaternion
            if (P == 0) return GMS_OK;
            gms_pseudomesh_repose_args r;
            memset(&r, 0, sizeof(r));
            r.P = P; r.face = a->face; r.coeffs = a->coeffs; r.V = a->V; r.F = a->F; r.vertices = a->vertices; r.faces = a->faces;
            gms_points_args pa;
            memset(&pa, 0, sizeof(pa));
            pa.P = P; pa.eps = a->eps; pa.xyz = RL.xyz; pa.scaling_act = RL.scales; pa.rotation_act = RL.rots;
            return launch("points_bound_expand_fwd", K_EXP_FWD, 0, st, (P + GMS_PM_BLOCK - 1) / GMS_PM_BLOCK, GMS_PM_BLOCK, 0,
                          k_points_bound_expand_fwd, r, pa, a->settings.viewmatrix);
        });
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
    if (a->sh_adam && a->anomaly)
        return set_err(GMS_E_ARG, "gms_train_frame: anomaly and sh_adam exclude each other (the fused step would update features before the scan)%s%s");
    const FrameModel m = {a->V, a->F, a->K, a->M, a->vertices, a->faces, a->alpha_raw, a->scale_raw, a->features, a->opacity_raw, a->eps,
                          a->segments, a->n_segments, a->alpha_activation};
    int P, rc;
    if ((rc = frame_gaussian_count("gms_train_frame", m, &P))) return rc;
    if ((rc = frame_sh_check("gms_train_frame", a->settings.sh_degree, a->M))) return rc;
    const int W = a->settings.image_width, H = a->settings.image_height;
    if (a->workspace_bytes < gms_frame_workspace_bytes(P, W, H)) return set_err(GMS_E_ARG, "gms_train_frame: workspace too small%s%s");
    FrameLayout FL = frame_layout(aligned_base(a->workspace), P, W, H);
    gms_raster_outputs out = {FL.image, FL.radii, FL.invdepth, 0};
    std::vector<gms_expand_args> ea;
    gms_raster_inputs in;
    gms_raster_saved saved;
    if ((rc = mesh_expand_forward(m, FL.g.xyz, FL.g.scales, FL.g.rots, cuda_stream, &ea))) return rc;
    const FrameGaussians g = {P, a->M, FL.g.xyz, FL.g.scales, FL.g.rots, a->features, a->opacity_raw, FL.g.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    // sh_adam: the preprocess backward updates `features` in place; it is the frame's last reader of them (the expansion
    // backward below does not read them)
    if ((rc = frame_loss_backward(a, FL, in, saved, FL.d_xyz, a->d_color_sh, cuda_stream))) return rc;
    if (a->event_sh_ready) GMS_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(a->event_sh_ready), st));
    // expansion backward (vertex gradients are accumulated with atomics: the caller keeps d_vertices zeroed)
    if ((rc = mesh_expand_backward(ea, FL.d_xyz, FL.d_scales, FL.d_rots, a->d_vertices, a->d_alpha_raw, a->d_scale_raw, cuda_stream)))
        return rc;
    if ((rc = anomaly_hook(a->anomaly, a->anomaly_stages, GMS_ANOMALY_EXPAND_BWD,
                           {{a->d_vertices, 3 * (int64_t)a->V, GMS_ANOMALY_DVERTICES}, {a->d_alpha_raw, 3 * (int64_t)P, GMS_ANOMALY_DALPHA_RAW},
                            {a->d_scale_raw, (int64_t)P, GMS_ANOMALY_DSCALE_RAW}}, 0, st))) return rc;
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
    return launch("free_act_fwd", K_EXP_FWD, 0, st, (P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, k_free_act_fwd, P, cols,
                  scaling_raw, rotation_raw, eps, scales, rots);
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
    if (a->sh_adam && a->anomaly)
        return set_err(GMS_E_ARG, "gms_free_train_frame: anomaly and sh_adam exclude each other (the fused step would update features before the scan)%s%s");
    int rc;
    if ((rc = frame_sh_check("gms_free_train_frame", a->settings.sh_degree, a->M))) return rc;
    const int W = a->settings.image_width, H = a->settings.image_height;
    if (W <= 0 || H <= 0) return set_err(GMS_E_ARG, "gms_free_train_frame: bad image size%s%s");
    if (a->workspace_bytes < gms_frame_workspace_bytes(P, W, H)) return set_err(GMS_E_ARG, "gms_free_train_frame: workspace too small%s%s");
    FrameLayout FL = frame_layout(aligned_base(a->workspace), P, W, H);
    gms_raster_outputs out = {FL.image, FL.radii, FL.invdepth, 0};
    gms_raster_inputs in;
    gms_raster_saved saved;
    if ((rc = free_act_fwd(P, a->scale_cols, a->scaling_raw, a->rotation_raw, a->eps, FL.g.scales, FL.g.rots, st))) return rc;
    const FrameGaussians g = {P, a->M, a->xyz, FL.g.scales, FL.g.rots, a->features, a->opacity_raw, FL.g.opac};
    if ((rc = frame_raster_forward(g, &a->settings, &out, alloc, alloc_user, a->binning_capacity, a->n_host_mapped, cuda_stream, &in,
                                   &saved))) return rc;
    if ((rc = frame_loss_backward(a, FL, in, saved, a->d_xyz, nullptr, cuda_stream))) return rc;
    if (P > 0) {
        FreeActBwd b;
        b.P = P; b.cols = a->scale_cols; b.rotation_raw = a->rotation_raw; b.scales = FL.g.scales;
        b.d_scales = FL.d_scales; b.d_rots = FL.d_rots; b.d_m2d = FL.d_m2d; b.radii = FL.radii;
        b.d_scaling_raw = a->d_scaling_raw; b.d_rotation_raw = a->d_rotation_raw; b.accum = a->accum; b.denom = a->denom;
        b.counters = geom_layout(aligned_base(saved.geom), P).counters;
        if ((rc = launch("free_act_bwd", K_EXP_BWD, 0, st, (P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, k_free_act_bwd, b)))
            return rc;
        if ((rc = anomaly_hook(a->anomaly, a->anomaly_stages, GMS_ANOMALY_ACTIVATION_BWD,
                               {{a->d_scaling_raw, (int64_t)P * a->scale_cols, GMS_ANOMALY_DSCALING_RAW},
                                {a->d_rotation_raw, 4 * (int64_t)P, GMS_ANOMALY_DROTATION_RAW},
                                {a->accum, a->accum ? (int64_t)P : 0, GMS_ANOMALY_ACCUM}}, 0, st))) return rc;
    }
    if (a->num_rendered) *a->num_rendered = saved.num_rendered;
    return GMS_OK;
}

int gms_free_render_frame(const gms_free_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    return render_frame("gms_free_render_frame", a, alloc, alloc_user, cuda_stream,
        [&](int* P) {
            if (!free_model_ok(a->P, a->M, a->scale_cols, a->xyz, a->scaling_raw, a->rotation_raw, a->features, a->opacity_raw))
                return set_err(GMS_E_ARG, "gms_free_render_frame: need P >= 0, 1 <= M <= 16, scale_cols 2 or 3 and every model tensor%s%s");
            if (!aligned16(a->rotation_raw)) return set_err(GMS_E_ARG, "gms_free_render_frame: rotation_raw must be 16-byte aligned%s%s");
            *P = a->P;
            return GMS_OK;
        },
        [&](int P, const RenderLayout& RL, const float** xyz) {
            *xyz = a->xyz;
            return free_act_fwd(P, a->scale_cols, a->scaling_raw, a->rotation_raw, a->eps, RL.scales, RL.rots, st);
        });
}

// ------------------------------------------------------------------------------------------ gs_flame checkpoint render

size_t gms_flame_render_workspace_bytes(int32_t P, int32_t W, int32_t H) { return gms_render_workspace_bytes(P, W, H); }

int gms_flame_render_frame(const gms_flame_render_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    return render_frame("gms_flame_render_frame", a, alloc, alloc_user, cuda_stream,
        [&](int* P) {
            if (!a->vertices || !a->faces || !a->alpha || !a->scaling_log || !a->rotation_raw || !a->features || !a->opacity_raw)
                return set_err(GMS_E_ARG, "gms_flame_render_frame: model tensors required%s%s");
            if (a->F < 0 || a->K < 1 || a->V < 1 || a->M < 1 || a->M > 16 || (int64_t)a->F * a->K > INT32_MAX)
                return set_err(GMS_E_ARG, "gms_flame_render_frame: need F >= 0, K >= 1, V >= 1, 1 <= M <= 16 and F*K < 2^31%s%s");
            if (!aligned16(a->rotation_raw)) return set_err(GMS_E_ARG, "gms_flame_render_frame: rotation_raw must be 16-byte aligned%s%s");
            *P = a->F * a->K;
            return GMS_OK;
        },
        [&](int P, const RenderLayout& RL, const float**) {
            if (P == 0) return GMS_OK;
            return launch("flame_act", K_EXP_FWD, 0, st, (P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, k_flame_act, P, a->K,
                          a->alpha, a->faces, a->vertices, a->scaling_log, a->rotation_raw, RL.xyz, RL.scales, RL.rots);
        });
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
    DensifyScratch S = densify_scratch(aligned_base(a->scratch), P);
    DensifyPlanK k;
    k.P = P; k.cols = a->scale_cols; k.accum = a->accum; k.denom = a->denom; k.scaling_raw = a->scaling_raw; k.opacity_raw = a->opacity_raw;
    k.eps = a->eps; k.grad_threshold = a->grad_threshold; k.split_scale = a->split_scale; k.min_opacity = a->min_opacity;
    k.max_world_scale = a->max_world_scale; k.flags = S.flags; k.fate = a->fate;
    span_begin(K_MISC, st);
    const int rc = launch("densify_plan", -1, 0, st, (P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, k_densify_plan, k);
    if (rc) return rc;
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
    DensifyScratch S = densify_scratch(const_cast<void*>(aligned_base(const_cast<void*>(a->scratch))), a->P);
    DensifyApplyK k;
    k.P = a->P; k.cols = a->scale_cols; k.F = 3 * a->M; k.eps = a->eps; k.incl = S.incl;
    k.kept = r[1]; k.clones = r[2]; k.splits = r[3]; k.normals = a->normals;
    for (int t = 0; t < 3; t++) {
        const gms_free_set& s = a->src[t];
        const gms_free_set& d = a->dst[t];
        k.src[t] = {s.xyz, s.scaling, s.rotation, s.opacity, s.features};
        k.dst[t] = {d.xyz, d.scaling, d.rotation, d.opacity, d.features};
    }
    return launch("densify_apply", K_MISC, 0, st, (a->P + GMS_FREE_BLOCK - 1) / GMS_FREE_BLOCK, GMS_FREE_BLOCK, 0, k_densify_apply, k);
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
    KnnLayout L = knn_layout(aligned_base(a->scratch), P);
    span_begin(K_MISC, st);
    int rc;
    if ((rc = launch("knn_bounds", -1, 0, st, GMS_KNN_BOUNDS_BLOCKS, 256, 0, k_knn_bounds, P, a->points, L.part))) return rc;
    if ((rc = launch("knn_bounds_fold", -1, 0, st, 1, 256, 0, k_knn_bounds_fold, L.part, L.bounds))) return rc;
    if ((rc = launch("knn_morton", -1, 0, st, (P + 255) / 256, 256, 0, k_knn_morton, P, a->points, L.bounds, L.code, L.idx))) return rc;
    size_t tb = L.cub_bytes;
    GMS_CUDA(cub::DeviceRadixSort::SortPairs(L.cub, tb, L.code, L.code_s, L.idx, L.idx_s, P, 0, 30, st));
    if ((rc = launch("knn_gather", -1, 0, st, (P + 255) / 256, 256, 0, k_knn_gather, P, a->points, L.idx_s, L.sorted))) return rc;
    if ((rc = launch("knn_box_bounds", -1, 0, st, (nbox + 7) / 8, 256, 0, k_knn_box_bounds, P, nbox, L.sorted, L.blo, L.bhi))) return rc;
    if ((rc = launch("knn_search", -1, 0, st, nbox, GMS_KNN_BOX, 0, k_knn_search, P, nbox, L.sorted, L.blo, L.bhi, a->dist2))) return rc;
    span_end(st);
    return GMS_OK;
}

// ---- alpha shape and normals (gms_alpha.cuh)

struct GridLayout {
    GmsGridStats* part;                 // [GMS_GRID_STAT_BLOCKS] partial bounds and sums
    GmsGrid* grid;                      // [1] origin, 1 / cell size, mean
    uint64_t* key; uint64_t* key_s;     // [P] cell keys, unsorted / sorted
    uint32_t* idx; uint32_t* idx_s;     // [P] point indices, unsorted / sorted
    float4* p4;                         // [P] points in index order, w = index
    float4* sorted;                     // [P] points in key order, w = index
    void* cub; size_t cub_bytes;
};

static GridLayout grid_layout(char*& p, int Pn) {
    GridLayout L;
    L.part = carve<GmsGridStats>(p, GMS_GRID_STAT_BLOCKS);
    L.grid = carve<GmsGrid>(p, 1);
    L.key = carve<uint64_t>(p, Pn); L.key_s = carve<uint64_t>(p, Pn);
    L.idx = carve<uint32_t>(p, Pn); L.idx_s = carve<uint32_t>(p, Pn);
    L.p4 = carve<float4>(p, Pn); L.sorted = carve<float4>(p, Pn);
    L.cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, L.cub_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    Pn, 0, 3 * GMS_GRID_BITS);
    return L;
}

// bounds, mean, cell keys and the key-sorted points; the cub temp storage is L.cub
static int grid_build(const GridLayout& L, int P, const float* pts, double hmin, cudaStream_t st) {
    int rc;
    if ((rc = launch("grid_stats", -1, 0, st, GMS_GRID_STAT_BLOCKS, 256, 0, k_grid_stats, P, pts, L.part))) return rc;
    if ((rc = launch("grid_fold", -1, 0, st, 1, 256, 0, k_grid_fold, P, L.part, hmin, L.grid))) return rc;
    if ((rc = launch("grid_keys", -1, 0, st, (P + 255) / 256, 256, 0, k_grid_keys, P, pts, L.grid, L.key, L.idx, L.p4))) return rc;
    size_t tb = L.cub_bytes;
    GMS_CUDA(cub::DeviceRadixSort::SortPairs(L.cub, tb, L.key, L.key_s, L.idx, L.idx_s, P, 0, 3 * GMS_GRID_BITS, st));
    return launch("grid_gather", -1, 0, st, (P + 255) / 256, 256, 0, k_grid_gather, P, L.p4, L.idx_s, L.sorted);
}

struct AlphaLayout {
    GridLayout g;
    int32_t* alive;                     // [P] 0 for a duplicate of a lower index
    int64_t* n_all; int64_t* off_all;   // [P+1] 3-alpha list lengths / offsets
    int64_t* n_up; int64_t* off_up;     // [P+1] 2-alpha higher-index list lengths / offsets
    int64_t* fcount; int64_t* foff;     // [P+1] faces per lowest vertex / offsets
    int32_t* ref; int32_t* voff;        // [P+1] referenced flags / vertex rows
    size_t total;
};

static AlphaLayout alpha_layout(void* base, int P) {
    AlphaLayout L;
    char* p = reinterpret_cast<char*>(base);
    const int Pn = P > 0 ? P : 1;
    L.alive = carve<int32_t>(p, Pn);
    L.n_all = carve<int64_t>(p, Pn + 1); L.off_all = carve<int64_t>(p, Pn + 1);
    L.n_up = carve<int64_t>(p, Pn + 1); L.off_up = carve<int64_t>(p, Pn + 1);
    L.fcount = carve<int64_t>(p, Pn + 1); L.foff = carve<int64_t>(p, Pn + 1);
    L.ref = carve<int32_t>(p, Pn + 1); L.voff = carve<int32_t>(p, Pn + 1);
    L.g = grid_layout(p, Pn);
    size_t scan64 = 0, scan32 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan64, (int64_t*)nullptr, (int64_t*)nullptr, Pn + 1);
    cub::DeviceScan::ExclusiveSum(nullptr, scan32, (int32_t*)nullptr, (int32_t*)nullptr, Pn + 1);
    L.g.cub_bytes = std::max(L.g.cub_bytes, std::max(scan64, scan32));
    L.g.cub = p;
    p += align_up(L.g.cub_bytes);
    L.total = (size_t)(p - reinterpret_cast<char*>(base));
    return L;
}

int gms_alpha_shape(const gms_alpha_shape_args* a, gms_alloc_fn alloc, void* alloc_user, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || !alloc || !a->n_faces || !a->n_vertices || a->P < 0 || a->P == INT32_MAX || !(a->alpha > 0.0) || !isfinite(a->alpha) ||
        (a->P > 0 && !a->points))
        return set_err(GMS_E_ARG, "gms_alpha_shape: need non-null arguments, 0 <= P < INT32_MAX and a finite alpha > 0%s%s");
    *a->n_faces = 0; *a->n_vertices = 0;
    if (a->P == 0) return GMS_OK;
    const int P = a->P, nb = (P + 255) / 256;
    const double alpha = a->alpha, alpha2 = alpha * alpha;
    void* sbase = alloc(alloc_user, GMS_ALPHA_BUF_SCRATCH, alpha_layout(nullptr, P).total + 256);
    if (!sbase) return set_err(GMS_E_ALLOC, "gms_alpha_shape: scratch allocation failed%s%s");
    AlphaLayout L = alpha_layout(aligned_base(sbase), P);
    int rc;
    span_begin(K_MISC, st);
    if ((rc = grid_build(L.g, P, a->points, 3.0 * alpha * (1.0 + 1e-6), st))) return rc;
    if ((rc = launch("alpha_dedup", -1, 0, st, nb, 256, 0, k_alpha_dedup, P, L.g.key_s, L.g.sorted, L.alive))) return rc;
    const double r_all2 = 9.0 * alpha2 * (1.0 + 1e-9), r_up2 = 4.0 * alpha2 * (1.0 + 1e-9);
    GMS_CUDA(cudaMemsetAsync(L.n_all + P, 0, sizeof(int64_t), st));
    GMS_CUDA(cudaMemsetAsync(L.n_up + P, 0, sizeof(int64_t), st));
    if ((rc = launch("alpha_lists_count", -1, 0, st, nb, 256, 0, k_alpha_lists<true>, P, L.g.key_s, L.g.sorted, L.alive, r_all2, r_up2,
                     L.n_all, L.n_up, (const int64_t*)nullptr, (const int64_t*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr))) return rc;
    size_t tb = L.g.cub_bytes;
    GMS_CUDA(cub::DeviceScan::ExclusiveSum(L.g.cub, tb, L.n_all, L.off_all, P + 1, st));
    tb = L.g.cub_bytes;
    GMS_CUDA(cub::DeviceScan::ExclusiveSum(L.g.cub, tb, L.n_up, L.off_up, P + 1, st));
    int64_t tot[2];
    GMS_CUDA(cudaMemcpyAsync(&tot[0], L.off_all + P, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaMemcpyAsync(&tot[1], L.off_up + P, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaStreamSynchronize(st));                // host synchronisation 1: the list lengths
    if (tot[1] >= INT32_MAX) return set_err(GMS_E_ARG, "gms_alpha_shape: the 2-alpha neighbour lists exceed 2^31 entries%s%s");
    const size_t n_all = (size_t)std::max<int64_t>(tot[0], 1), n_up = (size_t)std::max<int64_t>(tot[1], 1);
    size_t seg_bytes = 0;
    cub::DeviceSegmentedSort::SortKeys(nullptr, seg_bytes, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n_up, P, L.off_up, L.off_up + 1);
    const size_t lists_bytes = align_up(n_all * 4) + 2 * align_up(n_up * 4) + align_up(seg_bytes) + 256;
    void* lbase = alloc(alloc_user, GMS_ALPHA_BUF_LISTS, lists_bytes);
    if (!lbase) return set_err(GMS_E_ALLOC, "gms_alpha_shape: neighbour list allocation failed%s%s");
    char* lp = reinterpret_cast<char*>(aligned_base(lbase));
    int32_t* all = carve<int32_t>(lp, n_all);
    int32_t* up = carve<int32_t>(lp, n_up);
    int32_t* up_s = carve<int32_t>(lp, n_up);
    void* seg_tmp = lp;
    if ((rc = launch("alpha_lists_fill", -1, 0, st, nb, 256, 0, k_alpha_lists<false>, P, L.g.key_s, L.g.sorted, L.alive, r_all2, r_up2,
                     (int64_t*)nullptr, (int64_t*)nullptr, (const int64_t*)L.off_all, (const int64_t*)L.off_up, all, up))) return rc;
    if (tot[1] > 0) GMS_CUDA(cub::DeviceSegmentedSort::SortKeys(seg_tmp, seg_bytes, (const int32_t*)up, up_s, (int)tot[1], P, L.off_up,
                                                                L.off_up + 1, st));
    GMS_CUDA(cudaMemsetAsync(L.ref, 0, sizeof(int32_t) * (P + 1), st));
    GMS_CUDA(cudaMemsetAsync(L.fcount + P, 0, sizeof(int64_t), st));
    const int fb = (P + GMS_ALPHA_WARPS - 1) / GMS_ALPHA_WARPS;
    if ((rc = launch("alpha_faces_count", -1, 0, st, fb, GMS_ALPHA_WARPS * 32, 0, k_alpha_faces<true>, P, (const float4*)L.g.p4,
                     (const int64_t*)L.off_all, (const int32_t*)all, (const int64_t*)L.off_up, (const int32_t*)up_s, alpha2, L.fcount, L.ref,
                     (const int64_t*)nullptr, (const int32_t*)nullptr, (int64_t*)nullptr))) return rc;
    tb = L.g.cub_bytes;
    GMS_CUDA(cub::DeviceScan::ExclusiveSum(L.g.cub, tb, L.fcount, L.foff, P + 1, st));
    tb = L.g.cub_bytes;
    GMS_CUDA(cub::DeviceScan::ExclusiveSum(L.g.cub, tb, L.ref, L.voff, P + 1, st));
    int64_t F = 0;
    int32_t V = 0;
    GMS_CUDA(cudaMemcpyAsync(&F, L.foff + P, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaMemcpyAsync(&V, L.voff + P, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GMS_CUDA(cudaStreamSynchronize(st));                // host synchronisation 2: the output sizes
    *a->n_faces = F; *a->n_vertices = V;
    if (F > 0) {
        int64_t* faces = reinterpret_cast<int64_t*>(alloc(alloc_user, GMS_ALPHA_BUF_FACES, sizeof(int64_t) * 3 * (size_t)F));
        int64_t* index = reinterpret_cast<int64_t*>(alloc(alloc_user, GMS_ALPHA_BUF_INDEX, sizeof(int64_t) * (size_t)V));
        if (!faces || !index) return set_err(GMS_E_ALLOC, "gms_alpha_shape: output allocation failed%s%s");
        if ((rc = launch("alpha_faces_emit", -1, 0, st, fb, GMS_ALPHA_WARPS * 32, 0, k_alpha_faces<false>, P, (const float4*)L.g.p4,
                         (const int64_t*)L.off_all, (const int32_t*)all, (const int64_t*)L.off_up, (const int32_t*)up_s, alpha2,
                         (int64_t*)nullptr, (int32_t*)nullptr, (const int64_t*)L.foff, (const int32_t*)L.voff, faces))) return rc;
        if ((rc = launch("alpha_index", -1, 0, st, nb, 256, 0, k_alpha_index, P, (const int32_t*)L.ref, (const int32_t*)L.voff, index))) return rc;
    }
    span_end(st);
    return GMS_OK;
}

static size_t normals_layout(void* base, int P, GridLayout* out) {
    char* p = reinterpret_cast<char*>(base);
    GridLayout L = grid_layout(p, P > 0 ? P : 1);
    L.cub = p;
    p += align_up(L.cub_bytes);
    if (out) *out = L;
    return (size_t)(p - reinterpret_cast<char*>(base));
}

size_t gms_normals_scratch_bytes(int32_t P) { return normals_layout(nullptr, P, nullptr) + 512; }

int gms_estimate_normals(const gms_normals_args* a, void* cuda_stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (!a || a->P < 0 || !(a->radius > 0.0) || !isfinite(a->radius) || a->max_nn < 1 || a->max_nn > GMS_NORMALS_MAX_NN)
        return set_err(GMS_E_ARG, "gms_estimate_normals: need P >= 0, a finite radius > 0 and 1 <= max_nn <= GMS_NORMALS_MAX_NN%s%s");
    if (a->P == 0) return GMS_OK;
    if (!a->points || !a->normals || !a->scratch) return set_err(GMS_E_ARG, "gms_estimate_normals: null argument%s%s");
    if (a->scratch_bytes < gms_normals_scratch_bytes(a->P)) return set_err(GMS_E_ARG, "gms_estimate_normals: scratch too small%s%s");
    const int P = a->P;
    GridLayout L;
    normals_layout(aligned_base(a->scratch), P, &L);
    int rc;
    span_begin(K_MISC, st);
    if ((rc = grid_build(L, P, a->points, a->radius * (1.0 + 1e-6), st))) return rc;
    if ((rc = launch("normals", -1, 0, st, (P + 127) / 128, 128, 0, k_normals, P, (const uint64_t*)L.key_s, (const float4*)L.sorted,
                     (const float4*)L.p4, (const GmsGrid*)L.grid, a->radius * a->radius, (int)a->max_nn, a->normals))) return rc;
    span_end(st);
    return GMS_OK;
}

// ------------------------------------------------------------------------------------------ FLAME linear blend skinning

size_t gms_flame_lbs_workspace_bytes(int32_t V) {
    if (V <= 0) return 0;
    return gms_flame_ws(nullptr, V).floats * sizeof(float) + 256;
}

static int flame_lbs_check(const gms_flame_lbs_args* a, bool backward) {
    if (!a) return set_err(GMS_E_ARG, "gms_flame_lbs: null argument%s%s");
    if (a->V <= 0 || a->n_shape < 0 || a->n_shape > 300 || a->n_exp < 0 || a->n_exp > 100)
        return set_err(GMS_E_ARG, "gms_flame_lbs: need V > 0, 0 <= n_shape <= 300, 0 <= n_exp <= 100%s%s");
    if (a->n_joints != GMS_FLAME_NJ || a->parents[0] != -1)
        return set_err(GMS_E_ARG, "gms_flame_lbs: need 5 joints with parents[0] = -1%s%s");
    for (int j = 1; j < GMS_FLAME_NJ; j++)
        if (a->parents[j] < 0 || a->parents[j] >= j) return set_err(GMS_E_ARG, "gms_flame_lbs: need 0 <= parents[j] < j%s%s");
    const int B = a->n_shape + a->n_exp;
    const void* need[] = {a->v_template, a->posedirs, a->J_regressor, a->lbs_weights, a->pose, a->neck_pose, a->transl,
                          a->enlargement, a->workspace};
    for (const void* p : need)
        if (!p || (reinterpret_cast<size_t>(p) & 3)) return set_err(GMS_E_ARG, "gms_flame_lbs: null or misaligned pointer%s%s");
    const void* opt[] = {a->shapedirs, a->shape, a->expression, a->vertices_grad};
    for (const void* p : opt)
        if (reinterpret_cast<size_t>(p) & 3) return set_err(GMS_E_ARG, "gms_flame_lbs: misaligned pointer%s%s");
    if ((B > 0 && !a->shapedirs) || (a->n_shape > 0 && !a->shape) || (a->n_exp > 0 && !a->expression))
        return set_err(GMS_E_ARG, "gms_flame_lbs: null shape or expression pointer%s%s");
    if (a->workspace_bytes < gms_flame_lbs_workspace_bytes(a->V)) return set_err(GMS_E_ARG, "gms_flame_lbs: workspace too small%s%s");
    if (!backward) {
        if (!a->vertices || (reinterpret_cast<size_t>(a->vertices) & 3)) return set_err(GMS_E_ARG, "gms_flame_lbs: null or misaligned vertices%s%s");
        return GMS_OK;
    }
    float* const g[] = {a->d_pose, a->d_neck_pose, a->d_transl, a->d_enlargement, a->vertices_grad};
    for (float* p : g)
        if (!p || (reinterpret_cast<size_t>(p) & 3)) return set_err(GMS_E_ARG, "gms_flame_lbs: null or misaligned gradient pointer%s%s");
    if ((a->n_shape > 0 && (!a->d_shape || (reinterpret_cast<size_t>(a->d_shape) & 3))) ||
        (a->n_exp > 0 && (!a->d_expression || (reinterpret_cast<size_t>(a->d_expression) & 3))))
        return set_err(GMS_E_ARG, "gms_flame_lbs: null or misaligned shape / expression gradient%s%s");
    return GMS_OK;
}

int gms_flame_lbs_forward(const gms_flame_lbs_args* a, void* cuda_stream) {
    int rc = flame_lbs_check(a, false);
    if (rc != GMS_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    const int V = a->V;
    const int nsb = (V + GMS_FLAME_SB - 1) / GMS_FLAME_SB, nvb = (V + GMS_FLAME_VB - 1) / GMS_FLAME_VB;
    GmsFlameWs w = gms_flame_ws(reinterpret_cast<float*>(aligned_base(a->workspace)), V);
    GmsFlameParents par;
    for (int j = 0; j < GMS_FLAME_NJ; j++) par.p[j] = a->parents[j];
    span_begin(K_MISC, st);
    if ((rc = launch("flame_shape", -1, 0, st, nsb, 3 * GMS_FLAME_SB, 0, k_flame_shape, V, a->n_shape, a->n_exp, a->v_template, a->shapedirs,
                     a->shape, a->expression, a->J_regressor, w.vs, w.jpart))) return rc;
    if ((rc = launch("flame_joints", -1, 0, st, 1, 128, 0, k_flame_joints, nsb, w.jpart, a->pose, a->neck_pose, par, w.J, w.state))) return rc;
    if ((rc = launch("flame_skin", -1, 0, st, nvb, GMS_FLAME_VB, 0, k_flame_skin, V, w.vs, a->posedirs, a->lbs_weights, a->transl,
                     a->enlargement, w.state, w.vp, a->vertices, a->vertices_grad))) return rc;
    span_end(st);
    return GMS_OK;
}

int gms_flame_lbs_backward(const gms_flame_lbs_args* a, void* cuda_stream) {
    int rc = flame_lbs_check(a, true);
    if (rc != GMS_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    const int V = a->V, B = a->n_shape + a->n_exp;
    const int nvb = (V + GMS_FLAME_VB - 1) / GMS_FLAME_VB;
    GmsFlameWs w = gms_flame_ws(reinterpret_cast<float*>(aligned_base(a->workspace)), V);
    GmsFlameParents par;
    for (int j = 0; j < GMS_FLAME_NJ; j++) par.p[j] = a->parents[j];
    span_begin(K_MISC, st);
    if ((rc = launch("flame_skin_bwd", -1, 0, st, nvb, GMS_FLAME_VB, 0, k_flame_skin_bwd, V, w.vp, a->posedirs, a->lbs_weights, a->transl,
                     a->enlargement, w.state, a->vertices_grad, a->d_enlargement, w.dvp, w.bpart))) return rc;
    if ((rc = launch("flame_joints_bwd", -1, 0, st, 1, 128, 0, k_flame_joints_bwd, nvb, w.bpart, a->pose, a->neck_pose, par, w.J, w.state,
                     a->d_pose, a->d_neck_pose, a->d_transl, w.dJ))) return rc;
    if (B > 0 && (rc = launch("flame_betas_bwd", -1, 0, st, B, GMS_FLAME_CB, 0, k_flame_betas_bwd, V, a->n_shape, a->shapedirs,
                              a->J_regressor, w.dvp, w.dJ, a->d_shape, a->d_expression))) return rc;
    span_end(st);
    return GMS_OK;
}

int gms_nan_scan(const gms_nan_scan_args* a, void* cuda_stream) {
    if (!a || !a->record) return set_err(GMS_E_ARG, "gms_nan_scan: null record%s%s");
    if (a->n_buffers < 0 || a->n_buffers > GMS_NAN_SCAN_MAX_BUFFERS)
        return set_err(GMS_E_ARG, "gms_nan_scan: n_buffers must be 0..GMS_NAN_SCAN_MAX_BUFFERS%s%s");
    if (a->stage < 0 || a->stage >= GMS_ANOMALY_STAGES) return set_err(GMS_E_ARG, "gms_nan_scan: stage out of range%s%s");
    for (int i = 0; i < a->n_buffers; i++) {
        const gms_nan_buffer& b = a->buffers[i];
        if (b.n < 0 || b.n >= ((int64_t)1 << 48)) return set_err(GMS_E_ARG, "gms_nan_scan: a buffer needs 0 <= n < 2^48%s%s");
        if (b.tensor < 0 || b.tensor > 255) return set_err(GMS_E_ARG, "gms_nan_scan: tensor id out of range 0..255%s%s");
        if (b.n > 0 && (!b.ptr || (reinterpret_cast<size_t>(b.ptr) & 3)))
            return set_err(GMS_E_ARG, "gms_nan_scan: a non-empty buffer needs a 4-byte-aligned pointer%s%s");
    }
    return nan_scan_launch(a->stage, a->buffers, a->n_buffers, a->record, 0, reinterpret_cast<cudaStream_t>(cuda_stream));
}

}  // extern "C"
