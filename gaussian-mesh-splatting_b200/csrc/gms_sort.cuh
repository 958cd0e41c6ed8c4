// gms_sort.cuh -- hand-written stable LSD radix sort of (u32 key, u32 value) pairs for the tile binning, sm_90a.
//
// Replaces [upstream rasterizer_impl.cu: cub::DeviceRadixSort::SortPairs] -- and, unlike a library sort, takes the
// number of items from DEVICE memory (grid sized for a capacity, the count clamped to it, surplus CTAs exit), which is what a sync-free /
// graph-captured frame needs.  Two uses per frame (DESIGN.md section 3.3):
//   * the P Gaussians by depth bits (4 passes of 8 bits; pass 1 generates value = index on the fly),
//   * the N duplicates by tile id   (ceil(log2 T) = 13 bits at 1080p: one 8-bit and one 5-bit pass).
// Stability is what makes the result identical to the stock (tile << 32 | depth) sort: ties keep emission order.
//
// 3 launches per pass:
//   k_rs_hist     CTA tile = 256 threads x 16 items; shared-memory digit histogram -> hist[digit][cta]
//   k_rs_scan     one CTA per digit: exclusive scan of its row over CTAs (+ row total); the last CTA to finish scans the
//                 <= 256 totals into digit bases; also zeroes the next pass's histogram
//   k_rs_scatter  reloads the tile warp-striped (order inside a warp = (row, lane)), ranks every item among the
//                 equal-digit items before it with match.any + popc against per-warp running counters (one
//                 warp-aggregated shared atomic per distinct digit per row), turns the per-warp counts into CTA-local
//                 offsets, and writes key/value to  base[d] + row[d][cta] + local rank; while doing so it counts the
//                 item's NEXT digit into the histogram row of the CTA tile it lands in (no separate histogram pass).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define GMS_RS_THREADS 256
#define GMS_RS_ITEMS 16
#define GMS_RS_TILE (GMS_RS_THREADS * GMS_RS_ITEMS)      // 4096 items per CTA
#define GMS_RS_RADIX 256

__global__ void __launch_bounds__(GMS_RS_THREADS)
k_rs_hist(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ d_n, uint32_t capacity, int shift, uint32_t mask, int ncta,
          uint32_t* __restrict__ hist /* [RADIX][ncta] */, uint32_t* __restrict__ tickets /* [4], zeroed by the first pass */) {
    __shared__ uint32_t s_h[GMS_RS_RADIX];
    if (blockIdx.x == 0 && threadIdx.x < 4 && shift == 0) tickets[threadIdx.x] = 0;   // one ticket per pass, reset by the first pass
    const uint32_t n = min(*d_n, capacity);
    const uint32_t base = blockIdx.x * GMS_RS_TILE;
    const int lane = threadIdx.x & 31;
    s_h[threadIdx.x] = 0;
    __syncthreads();
    if (base < n) {
        uint32_t key[GMS_RS_ITEMS];
#pragma unroll
        for (int i = 0; i < GMS_RS_ITEMS; i++) {
            const uint32_t k = base + i * GMS_RS_THREADS + threadIdx.x;
            key[i] = k < n ? keys[k] : 0xFFFFFFFFu;
        }
#pragma unroll
        for (int i = 0; i < GMS_RS_ITEMS; i++) {
            const uint32_t k = base + i * GMS_RS_THREADS + threadIdx.x;
            const bool ok = k < n;
            const uint32_t d = ok ? ((key[i] >> shift) & mask) : 0xFFFFu;
            const uint32_t peers = __match_any_sync(0xffffffffu, d);          // warp-aggregated: one atomic per distinct digit
            if (ok && (peers & ((1u << lane) - 1u)) == 0) atomicAdd(&s_h[d], (uint32_t)__popc(peers));
        }
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * ncta + blockIdx.x] = s_h[threadIdx.x];
}

// one CTA per digit: exclusive scan of hist[d][0..ncta) in place, total -> totals[d]; zeroes the same row of the NEXT
// pass's histogram (filled by this pass's scatter); the last CTA to finish turns the 256 totals into digit bases.
__global__ void __launch_bounds__(256) k_rs_scan(uint32_t* __restrict__ hist, int ncta, uint32_t* __restrict__ totals,
                                                 uint32_t* __restrict__ bases, uint32_t* __restrict__ ticket,
                                                 uint32_t* __restrict__ hist_next) {
    __shared__ uint32_t s_w[8];
    __shared__ uint32_t s_carry;
    __shared__ bool s_last;
    uint32_t* row = hist + (size_t)blockIdx.x * ncta;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int c0 = 0; c0 < ncta; c0 += 256) {
        const int c = c0 + threadIdx.x;
        const uint32_t v = c < ncta ? row[c] : 0u;
        if (hist_next && c < ncta) hist_next[(size_t)blockIdx.x * ncta + c] = 0u;
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        if (lane == 31) s_w[warp] = x;
        __syncthreads();
        uint32_t wbase = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) if (w < warp) wbase += s_w[w];
        const uint32_t carry = s_carry;
        if (c < ncta) row[c] = carry + wbase + x - v;
        __syncthreads();
        if (threadIdx.x == 255) s_carry = carry + wbase + x;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        totals[blockIdx.x] = s_carry;
        __threadfence();
        s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const uint32_t v = *reinterpret_cast<volatile uint32_t*>(totals + threadIdx.x);
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    uint32_t wbase = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) if (w < warp) wbase += s_w[w];
    bases[threadIdx.x] = wbase + x - v;
}

__global__ void __launch_bounds__(GMS_RS_THREADS, 3)
k_rs_scatter(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in /* NULL: value = index */,
             const uint32_t* __restrict__ d_n, uint32_t capacity, int shift, uint32_t mask, int ncta, const uint32_t* __restrict__ hist,
             const uint32_t* __restrict__ bases, uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
             uint32_t* __restrict__ hist_next /* NULL on the last pass */, int next_shift, uint32_t next_mask) {
    __shared__ uint32_t s_cnt[8][GMS_RS_RADIX];     // per-warp running digit counts, then CTA-local warp offsets
    __shared__ uint32_t s_gbase[GMS_RS_RADIX];      // global offset of this CTA's first item of each digit
    const uint32_t n = min(*d_n, capacity);
    const uint32_t cta_base = blockIdx.x * GMS_RS_TILE;
    if (cta_base >= n) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int w = 0; w < 8; w++) s_cnt[w][threadIdx.x] = 0;
    s_gbase[threadIdx.x] = bases[threadIdx.x] + hist[(size_t)threadIdx.x * ncta + blockIdx.x];
    __syncthreads();
    // warp `warp` owns items [wbase, wbase + 32*ITEMS), row i = items wbase + 32 i + lane  (order = (i, lane))
    const uint32_t wbase = cta_base + warp * (32 * GMS_RS_ITEMS);
    uint32_t key[GMS_RS_ITEMS], rank[GMS_RS_ITEMS];
    const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
    for (int i = 0; i < GMS_RS_ITEMS; i++) {
        const uint32_t k = wbase + i * 32 + lane;
        key[i] = k < n ? keys_in[k] : 0xFFFFFFFFu;
    }
    // Row i of the warp: equal-digit lanes find each other with match.any; the lowest of them bumps the warp's running
    // counter with ONE shared-memory atomic whose return value is the count of that digit in rows < i (atomics of one
    // warp to one address retire in program order), and hands it to its peers with a shuffle.  No barrier between rows,
    // so the 16 rows overlap in the pipeline.
#pragma unroll
    for (int i = 0; i < GMS_RS_ITEMS; i++) {
        const uint32_t k = wbase + i * 32 + lane;
        const bool ok = k < n;
        const uint32_t d = ok ? ((key[i] >> shift) & mask) : 0xFFFFu;     // out-of-range items never match a real digit
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t before = 0;
        if (ok && lane == leader) before = atomicAdd(&s_cnt[warp][d], (uint32_t)__popc(peers));
        before = __shfl_sync(0xffffffffu, before, leader);
        rank[i] = before + __popc(peers & lt);
    }
    __syncthreads();
    {   // per digit: exclusive scan over the 8 warps -> warp offsets inside the CTA
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) { const uint32_t c = s_cnt[w][threadIdx.x]; s_cnt[w][threadIdx.x] = run; run += c; }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < GMS_RS_ITEMS; i++) {
        const uint32_t k = wbase + i * 32 + lane;
        const bool ok = k < n;
        uint32_t pos = 0, d = 0;
        if (ok) {
            d = (key[i] >> shift) & mask;
            pos = s_gbase[d] + s_cnt[warp][d] + rank[i];
            keys_out[pos] = key[i];
            vals_out[pos] = vals_in ? vals_in[k] : k;
        }
        if (hist_next) {
            // The item now lives in CTA tile pos / 4096 of the next pass: count its next digit there (saves a pass over the
            // keys).  Lanes of the row that agree on (next digit, tile) -- nearly all of them when the next digit is
            // constant, e.g. the exponent byte of the depth keys -- are merged into one global atomic.
            const uint32_t slot = ok ? ((key[i] >> next_shift) & next_mask) * (uint32_t)ncta + pos / GMS_RS_TILE : 0xFFFFFFFFu;
            const uint32_t peers = __match_any_sync(0xffffffffu, slot);
            if (ok && (peers & lt) == 0) atomicAdd(&hist_next[slot], (uint32_t)__popc(peers));
        }
    }
}

static inline size_t gms_sort_temp_bytes(int64_t capacity) {
    const size_t ncta = (size_t)((capacity + GMS_RS_TILE - 1) / GMS_RS_TILE) + 1;
    return (2 * GMS_RS_RADIX * ncta + 2 * GMS_RS_RADIX + 64) * sizeof(uint32_t) + 512;
}

// Sorts min(*d_n, capacity) pairs by key bits [0, nbits).  The clamp keeps an overflowed sync-free frame (device N above
// the capacity its buffers were sized for) inside those buffers; such a frame renders the background anyway.  Only the
// first min(*d_n, capacity) entries of any buffer are written.  Ping-pongs between (k0,v0) and (k1,v1); the first pass reads
// (keys_src, vals_src) where vals_src may be NULL (value = index).  Returns which buffer holds the result (0 or 1), or -1
// on launch failure.
static int gms_radix_sort_pairs(const uint32_t* keys_src, const uint32_t* vals_src, uint32_t* k0, uint32_t* v0, uint32_t* k1,
                                uint32_t* v1, const uint32_t* d_n, int64_t capacity, int nbits, void* temp, cudaStream_t st,
                                int64_t* launches) {
    const int ncta = (int)((capacity + GMS_RS_TILE - 1) / GMS_RS_TILE);
    if (ncta <= 0) return 0;
    const uint32_t cap32 = (uint32_t)(capacity > 0xFFFFFFFFll ? 0xFFFFFFFFll : capacity);
    uint32_t* histA = reinterpret_cast<uint32_t*>(temp);
    uint32_t* histB = histA + (size_t)GMS_RS_RADIX * (ncta + 1);
    uint32_t* totals = histB + (size_t)GMS_RS_RADIX * (ncta + 1);
    uint32_t* bases = totals + GMS_RS_RADIX;
    uint32_t* tickets = bases + GMS_RS_RADIX;
    const uint32_t* kin = keys_src; const uint32_t* vin = vals_src;
    int dst = 0, pass = 0;
    for (int shift = 0; shift < nbits; shift += 8, pass++) {
        const int bits = nbits - shift < 8 ? nbits - shift : 8;
        const uint32_t mask = (1u << bits) - 1u;
        uint32_t* ko = dst ? k1 : k0; uint32_t* vo = dst ? v1 : v0;
        // hist_next stays NULL: the digits of each pass are counted by this separate shared-memory histogram pass, not inside
        // the previous pass's scatter with global atomics.
        k_rs_hist<<<ncta, GMS_RS_THREADS, 0, st>>>(kin, d_n, cap32, shift, mask, ncta, histA, tickets);
        k_rs_scan<<<GMS_RS_RADIX, 256, 0, st>>>(histA, ncta, totals, bases, tickets + pass, nullptr);
        k_rs_scatter<<<ncta, GMS_RS_THREADS, 0, st>>>(kin, vin, d_n, cap32, shift, mask, ncta, histA, bases, ko, vo, nullptr, 0, 0u);
        if (launches) *launches += 3;
        if (cudaGetLastError() != cudaSuccess) return -1;
        kin = ko; vin = vo;
        dst ^= 1;
    }
    return dst ^ 1;
}
