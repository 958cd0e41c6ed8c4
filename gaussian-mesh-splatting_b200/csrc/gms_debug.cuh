// gms_debug.cuh -- the binning check of debug mode (gms_debug_check_bins, and every one-call frame run with settings.debug).
//
// The composite kernels trust four invariants of the binned point list and do not test them: the list is in (tile, depth
// key) order, the tile ranges partition it by tile, every entry's Gaussian covers its tile, and every survivor list of a
// quad points into its tile's range in ascending order.  Under debug a frame checks them on its own buffers:
//
//   k_debug_ranges  one CTA walks the T ranges in tile order (a block scan carries the end of the last non-empty range):
//                   each range lies in [0, n), a non-empty one starts where the previous non-empty one ended, the last
//                   ends at n                                                                               -> check 2
//   k_debug_list    one warp per tile walks the tile's entries: the tile key (when the path keeps keys) is the tile
//                   (check 2), the Gaussian index is < P with radii > 0 and a rectangle holding the tile (check 3), the
//                   (depth key, index) pair is strictly greater than the previous entry's (check 1).  The same grid adds up
//                   the tile rectangles of the Gaussians with radii > 0: with no duplicates in a tile (check 1) and every
//                   entry inside its Gaussian's rectangle (check 3), that sum equals n exactly when each range holds all
//                   the entries of its tile (the host compares the two)
//   k_debug_surv    one warp per (tile, quad): at most `range length` survivors, each < the range length, strictly
//                   ascending                                                                               -> check 4
//
// Every read is bounds-checked against n, P and T, so a corrupt list cannot make the check fault.  A violation is recorded
// as the key check << 56 | index, kept at its smallest (atomicMin), as gms_nan_scan keys its NaNs; per check, the Gaussian
// and the tile of the smallest index ride along in index << 32 | value words.  A clean list writes nothing but `n`.
#pragma once
#include <stdint.h>
#include <cub/block/block_scan.cuh>

#define GMS_DBG_BLOCK 256
#define GMS_DBG_RANGES_BLOCK 1024
#define GMS_DBG_NONE 0xFFFFFFFFu            // no tile / no Gaussian in a detail word

struct GmsBinRecord {
    unsigned long long key;                 // check << 56 | index, smallest; ~0: clean
    unsigned long long gid[5];              // [check] index << 32 | Gaussian of the smallest index
    unsigned long long tile[5];             // [check] index << 32 | tile of the smallest index
    unsigned long long area;                // sum of the tile rectangles of the Gaussians with radii > 0
    unsigned long long n;                   // the list length checked; ~0 after an overflowed frame (no list)
};

struct GmsBinCheck {
    int P, T, gx;
    int64_t n;                              // list length, when d_n is NULL
    const uint32_t* d_n;                    // device (N, overflow flag) of a frame, or NULL
    int64_t cap;                            // entries the list buffers hold
    const uint32_t* point_list;             // [cap] Gaussian indices
    const void* keys;                       // [cap] tile keys (uint16 when key16, else uint32), or NULL
    int key16;
    const int2* ranges;                     // [T]
    const int32_t* radii;                   // [P]
    const uint2* rect;                      // [P] x0 | y0 << 16, x1 | y1 << 16
    const uint32_t* dkey;                   // [P] depth keys
    const uint32_t* surv;                   // [4 cap] per-quad survivor lists, or NULL
    const uint32_t* nsurv;                  // [4T]
    GmsBinRecord* rec;
};

// The list length the check walks: n, or the frame's device N; -1 when the frame overflowed (every range must be empty).
__device__ __forceinline__ int64_t gms_dbg_len(const GmsBinCheck& c) {
    if (!c.d_n) return c.n;
    const uint32_t N = c.d_n[0];
    return (c.d_n[1] || (int64_t)N > c.cap) ? -1 : (int64_t)N;
}

__device__ __forceinline__ void gms_dbg_flag(GmsBinRecord* r, int check, uint64_t index, uint32_t tile, uint32_t gid) {
    atomicMin(&r->key, (unsigned long long)check << 56 | index);
    atomicMin(&r->gid[check], (unsigned long long)(index << 32) | gid);
    atomicMin(&r->tile[check], (unsigned long long)(index << 32) | tile);
}

struct GmsMaxInt { __device__ int operator()(int a, int b) const { return a > b ? a : b; } };

__global__ void __launch_bounds__(GMS_DBG_RANGES_BLOCK) k_debug_ranges(GmsBinCheck c) {
    using Scan = cub::BlockScan<int, GMS_DBG_RANGES_BLOCK>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int s_end;
    const int64_t len = gms_dbg_len(c);
    const int64_t n = len < 0 ? 0 : len;
    if (threadIdx.x == 0) { s_end = 0; c.rec->n = len < 0 ? ~0ull : (unsigned long long)len; }
    __syncthreads();
    for (int t0 = 0; t0 < c.T; t0 += GMS_DBG_RANGES_BLOCK) {
        const int t = t0 + threadIdx.x;
        const bool in = t < c.T;
        const int2 r = in ? c.ranges[t] : make_int2(0, 0);
        const bool full = in && r.y > r.x;
        const int carry = s_end;
        int before, agg;
        Scan(tmp).ExclusiveScan(full ? r.y : 0, before, carry, GmsMaxInt(), agg);
        if (in && (r.x < 0 || r.y < r.x || (int64_t)r.y > n || (full && r.x != before)))
            gms_dbg_flag(c.rec, 2, (uint64_t)(r.x < 0 ? 0 : r.x), (uint32_t)t, GMS_DBG_NONE);
        __syncthreads();
        if (threadIdx.x == 0) s_end = agg > carry ? agg : carry;
        __syncthreads();
    }
    if (threadIdx.x == 0 && (int64_t)s_end != n) gms_dbg_flag(c.rec, 2, (uint64_t)s_end, GMS_DBG_NONE, GMS_DBG_NONE);
}

__global__ void __launch_bounds__(GMS_DBG_BLOCK, 1) k_debug_list(GmsBinCheck c) {
    const int64_t n = gms_dbg_len(c);
    const int lane = threadIdx.x & 31;
    // 32-bit strides (P < 2^31; T <= 2^26, so the grid of T warps holds fewer than 2^31 threads): no 64-bit division for the
    // trip counts
    const int nthreads = (int)gridDim.x * GMS_DBG_BLOCK;
    unsigned long long area = 0;
    for (int g = (int)blockIdx.x * GMS_DBG_BLOCK + (int)threadIdx.x; g < c.P; g += nthreads) {
        const uint2 q = c.rect[g];
        const int w = (int)(q.y & 0xFFFFu) - (int)(q.x & 0xFFFFu), h = (int)(q.y >> 16) - (int)(q.x >> 16);
        if (c.radii[g] > 0 && w > 0 && h > 0) area += (unsigned long long)w * (unsigned long long)h;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) area += __shfl_xor_sync(0xffffffffu, area, o);
    if (lane == 0 && area) atomicAdd(&c.rec->area, area);
    const int nwarps = nthreads >> 5;
    for (int t = ((int)blockIdx.x * GMS_DBG_BLOCK + (int)threadIdx.x) >> 5; t < c.T; t += nwarps) {
        const int2 r = c.ranges[t];
        if (r.x < 0 || r.y <= r.x || (int64_t)r.y > n) continue;     // empty, or reported by k_debug_ranges
        const uint32_t ty = (uint32_t)t / (uint32_t)c.gx, tx = (uint32_t)t - ty * (uint32_t)c.gx;
        for (int j = r.x + lane; j < r.y; j += 32) {
            const uint32_t g = c.point_list[j];
            if (c.keys) {
                const uint32_t k = c.key16 ? (uint32_t)static_cast<const uint16_t*>(c.keys)[j] : static_cast<const uint32_t*>(c.keys)[j];
                if (k != (uint32_t)t) gms_dbg_flag(c.rec, 2, (uint64_t)j, (uint32_t)t, g);
            }
            if (g >= (uint32_t)c.P) { gms_dbg_flag(c.rec, 3, (uint64_t)j, (uint32_t)t, g); continue; }
            const uint2 q = c.rect[g];
            if (c.radii[g] <= 0 || tx < (q.x & 0xFFFFu) || tx >= (q.y & 0xFFFFu) || ty < (q.x >> 16) || ty >= (q.y >> 16))
                gms_dbg_flag(c.rec, 3, (uint64_t)j, (uint32_t)t, g);
            if (j > r.x) {
                const uint32_t p = c.point_list[j - 1];
                if (p < (uint32_t)c.P && ((uint64_t)c.dkey[p] << 32 | p) >= ((uint64_t)c.dkey[g] << 32 | g))
                    gms_dbg_flag(c.rec, 1, (uint64_t)j, (uint32_t)t, g);
            }
        }
    }
}

// index: the survivor's slot in `surv` (a quad whose count exceeds its range: the first slot past the quad's region)
__global__ void __launch_bounds__(GMS_DBG_BLOCK) k_debug_surv(GmsBinCheck c) {
    const int64_t n = gms_dbg_len(c);
    const int64_t w = ((int64_t)blockIdx.x * GMS_DBG_BLOCK + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= 4 * (int64_t)c.T) return;
    const int t = (int)(w >> 2), quad = (int)(w & 3);
    const int2 r = c.ranges[t];
    if (r.x < 0 || r.y < r.x || (int64_t)r.y > n) return;            // reported by k_debug_ranges
    const uint32_t len = (uint32_t)(r.y - r.x);
    const uint64_t base = 4 * (uint64_t)r.x + (uint64_t)quad * len;
    uint32_t cnt = c.nsurv[w];
    if (cnt > len) {
        if (lane == 0) gms_dbg_flag(c.rec, 4, base + len, (uint32_t)t, GMS_DBG_NONE);
        cnt = len;
    }
    for (uint32_t i = lane; i < cnt; i += 32) {
        const uint32_t s = c.surv[base + i];
        if (s >= len || (i > 0 && c.surv[base + i - 1] >= s))
            gms_dbg_flag(c.rec, 4, base + i, (uint32_t)t, s < len ? c.point_list[r.x + s] : GMS_DBG_NONE);
    }
}
