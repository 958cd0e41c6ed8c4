// gms_knn.cuh -- mean squared distance to the three nearest other points (simple-knn's distCUDA2), exact, sm_90a.
//
// Definition (the contract; include/gms_b200.h states it for callers):
//   d(q,p)   = (dx*dx + dy*dy) + dz*dz, dx = q.x - p.x, every operation one round-to-nearest fp32 op, never an FMA
//   b0 <= b1 <= b2: the three smallest d(points[i], points[j]) over j != i (tied values, duplicates at 0 included, count
//   separately);  dist2[i] = ((b0 + b1) + b2) / 3.
// The result depends on the multiset of distance values only, so neither the visit order below nor the launch
// configuration can change a bit of it.
//
// Algorithm (Morton boxes):
//   1. the bounding box of the cloud, reduced on the device in two passes;
//   2. a 30-bit Morton code per point from that box (an axis of zero extent gets code 0);
//   3. a stable radix sort of (code, index);
//   4. the sorted points gathered as float4 (x, y, z, original index);
//   5. per box of GMS_KNN_BOX consecutive sorted points, its min / max;
//   6. one CTA per box of queries (Morton-adjacent, so spatially compact): each thread seeds its top-3 from its own box,
//      then the CTA walks the other boxes outward in sort order, GMS_KNN_BOX of them per round.  A box is skipped for the
//      whole CTA when its lower bound to the CTA's query box exceeds the largest b2 of the CTA; a surviving box is staged
//      in shared memory and every thread scans it unless the box's lower bound to its own point exceeds its own b2.
//
// Why pruning is exact.  A lower bound is computed with the same round-to-nearest sequence as d: per axis the gap
// g = max(lo - q, q - hi, 0) (for box-to-box: max(lo_c - hi_q, lo_q - hi_c, 0)) by __fsub_rn, then squared and summed in
// d's order.  Round-to-nearest is monotone: for p in the box, p.x - q.x >= lo - q exactly, so fl(p.x - q.x) >= fl(lo - q),
// i.e. |dx| >= g; squares of non-negative values and sums of them are monotone too, so bound <= d for every point of the
// box.  A box is skipped only when bound > b2, strictly, so every skipped point has d > b2 and could not have entered the
// top-3 (an insertion needs d < b2).  b2 only decreases, so a bound checked against an earlier, larger b2 stays valid.
#pragma once
#include "gms_common.cuh"
#include "../../include/gms_b200.h"     // GMS_KNN_BOX: points per box = threads per search CTA

struct KnnBounds { float3 lo, hi; };

#define GMS_KNN_BOUNDS_BLOCKS 256

__device__ __forceinline__ void knn_bounds_add(KnnBounds& b, float x, float y, float z) {
    b.lo = make_float3(fminf(b.lo.x, x), fminf(b.lo.y, y), fminf(b.lo.z, z));
    b.hi = make_float3(fmaxf(b.hi.x, x), fmaxf(b.hi.y, y), fmaxf(b.hi.z, z));
}

// min / max over the CTA (256 threads) of each thread's bounds; thread 0 returns the result
__device__ __forceinline__ KnnBounds knn_bounds_cta(KnnBounds b) {
    __shared__ KnnBounds part[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        knn_bounds_add(b, __shfl_xor_sync(0xffffffffu, b.lo.x, o), __shfl_xor_sync(0xffffffffu, b.lo.y, o),
                       __shfl_xor_sync(0xffffffffu, b.lo.z, o));
        knn_bounds_add(b, __shfl_xor_sync(0xffffffffu, b.hi.x, o), __shfl_xor_sync(0xffffffffu, b.hi.y, o),
                       __shfl_xor_sync(0xffffffffu, b.hi.z, o));
    }
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = b;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < 8; w++) {
            knn_bounds_add(b, part[w].lo.x, part[w].lo.y, part[w].lo.z);
            knn_bounds_add(b, part[w].hi.x, part[w].hi.y, part[w].hi.z);
        }
    return b;
}

// Bounding box of the cloud in two passes: GMS_KNN_BOUNDS_BLOCKS partial boxes, then one CTA folds them.
__global__ void __launch_bounds__(256) k_knn_bounds(int P, const float* __restrict__ pts, KnnBounds* __restrict__ part) {
    KnnBounds b = {make_float3(INFINITY, INFINITY, INFINITY), make_float3(-INFINITY, -INFINITY, -INFINITY)};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x)
        knn_bounds_add(b, pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]);
    b = knn_bounds_cta(b);
    if (threadIdx.x == 0) part[blockIdx.x] = b;
}

__global__ void __launch_bounds__(256) k_knn_bounds_fold(const KnnBounds* __restrict__ part, KnnBounds* __restrict__ box) {
    KnnBounds b = part[threadIdx.x];
    b = knn_bounds_cta(b);
    if (threadIdx.x == 0) *box = b;
}

__device__ __forceinline__ uint32_t knn_spread10(uint32_t v) {      // 10 bits -> every third bit of 30
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

__device__ __forceinline__ uint32_t knn_cell(float x, float lo, float hi) {
    const float ext = hi - lo;
    if (!(ext > 0.f)) return 0u;
    // NaN (an infinite extent) maps to 0 through fmaxf; the code only orders the search, it never changes the result
    return (uint32_t)fminf(fmaxf((x - lo) / ext * 1024.f, 0.f), 1023.f);
}

__global__ void __launch_bounds__(256) k_knn_morton(int P, const float* __restrict__ pts, const KnnBounds* __restrict__ box,
                                                    uint32_t* __restrict__ code, uint32_t* __restrict__ idx) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const KnnBounds b = *box;
    const float* p = pts + 3 * (size_t)i;
    code[i] = knn_spread10(knn_cell(p[0], b.lo.x, b.hi.x)) << 2 | knn_spread10(knn_cell(p[1], b.lo.y, b.hi.y)) << 1 |
              knn_spread10(knn_cell(p[2], b.lo.z, b.hi.z));
    idx[i] = i;
}

__global__ void __launch_bounds__(256) k_knn_gather(int P, const float* __restrict__ pts, const uint32_t* __restrict__ idx,
                                                    float4* __restrict__ sorted) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const uint32_t i = idx[k];
    const float* p = pts + 3 * (size_t)i;
    sorted[k] = make_float4(p[0], p[1], p[2], __uint_as_float(i));
}

// One warp per box: min / max over its (up to) GMS_KNN_BOX sorted points.
__global__ void __launch_bounds__(256) k_knn_box_bounds(int P, int nbox, const float4* __restrict__ sorted, float4* __restrict__ blo,
                                                        float4* __restrict__ bhi) {
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= nbox) return;
    float3 lo = make_float3(INFINITY, INFINITY, INFINITY), hi = make_float3(-INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int k = lane; k < GMS_KNN_BOX; k += 32) {
        const int j = b * GMS_KNN_BOX + k;
        if (j < P) {
            const float4 v = sorted[j];
            lo = make_float3(fminf(lo.x, v.x), fminf(lo.y, v.y), fminf(lo.z, v.z));
            hi = make_float3(fmaxf(hi.x, v.x), fmaxf(hi.y, v.y), fmaxf(hi.z, v.z));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o)); hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o)); hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o)); hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
    }
    if (lane == 0) { blo[b] = make_float4(lo.x, lo.y, lo.z, 0.f); bhi[b] = make_float4(hi.x, hi.y, hi.z, 0.f); }
}

__device__ __forceinline__ float knn_sum3(float gx, float gy, float gz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz));
}

__device__ __forceinline__ float knn_d(const float4& q, const float4& p) {
    return knn_sum3(__fsub_rn(q.x, p.x), __fsub_rn(q.y, p.y), __fsub_rn(q.z, p.z));
}

// lower bound of d(q, p) over p in [lo, hi]
__device__ __forceinline__ float knn_point_box(const float4& q, const float4& lo, const float4& hi) {
    return knn_sum3(fmaxf(fmaxf(__fsub_rn(lo.x, q.x), __fsub_rn(q.x, hi.x)), 0.f),
                    fmaxf(fmaxf(__fsub_rn(lo.y, q.y), __fsub_rn(q.y, hi.y)), 0.f),
                    fmaxf(fmaxf(__fsub_rn(lo.z, q.z), __fsub_rn(q.z, hi.z)), 0.f));
}

// lower bound of d(q, p) over q in [qlo, qhi], p in [lo, hi]
__device__ __forceinline__ float knn_box_box(const float4& qlo, const float4& qhi, const float4& lo, const float4& hi) {
    return knn_sum3(fmaxf(fmaxf(__fsub_rn(lo.x, qhi.x), __fsub_rn(qlo.x, hi.x)), 0.f),
                    fmaxf(fmaxf(__fsub_rn(lo.y, qhi.y), __fsub_rn(qlo.y, hi.y)), 0.f),
                    fmaxf(fmaxf(__fsub_rn(lo.z, qhi.z), __fsub_rn(qlo.z, hi.z)), 0.f));
}

__device__ __forceinline__ void knn_insert(float d, float& b0, float& b1, float& b2) {
    if (d < b2) {
        if (d < b1) {
            b2 = b1;
            if (d < b0) { b1 = b0; b0 = d; } else { b1 = d; }
        } else {
            b2 = d;
        }
    }
}

__global__ void __launch_bounds__(GMS_KNN_BOX) k_knn_search(int P, int nbox, const float4* __restrict__ sorted,
                                                            const float4* __restrict__ blo, const float4* __restrict__ bhi,
                                                            float* __restrict__ dist2) {
    constexpr int B = GMS_KNN_BOX, NW = GMS_KNN_BOX / 32;
    __shared__ float4 stage[B];
    __shared__ int cand[B];
    __shared__ int ncand[NW];
    __shared__ uint32_t wmax[NW];
    const int box = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int i = box * B + t;
    const bool active = i < P;
    const float4 q = active ? sorted[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    stage[t] = q;
    __syncthreads();
    float b0 = INFINITY, b1 = INFINITY, b2 = INFINITY;
    const int nown = min(B, P - box * B);
    if (active)
        for (int j = 0; j < nown; j++)
            if (j != t) knn_insert(knn_d(q, stage[j]), b0, b1, b2);
    const float4 qlo = blo[box], qhi = bhi[box];
    const int reach = max(box, nbox - 1 - box);
    for (int r = 0; r * (B / 2) < reach; r++) {
        // the CTA's largest b2 (non-negative floats order as their bit patterns; inactive threads take no part)
        const uint32_t m = __reduce_max_sync(0xffffffffu, active ? __float_as_uint(b2) : 0u);
        if (lane == 0) wmax[w] = m;
        __syncthreads();
        uint32_t lim_bits = wmax[0];
#pragma unroll
        for (int k = 1; k < NW; k++) lim_bits = max(lim_bits, wmax[k]);
        const float lim = __uint_as_float(lim_bits);
        // this round's boxes: offsets r*B/2 + 1 .. (r+1)*B/2 on both sides, nearest first
        const int off = r * (B / 2) + (t >> 1) + 1;
        const int cb = (t & 1) ? box - off : box + off;
        const bool keep = cb >= 0 && cb < nbox && !(knn_box_box(qlo, qhi, blo[cb], bhi[cb]) > lim);
        const uint32_t bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) ncand[w] = __popc(bal);
        __syncthreads();
        int base = 0, total = 0;
#pragma unroll
        for (int k = 0; k < NW; k++) { base += k < w ? ncand[k] : 0; total += ncand[k]; }
        if (keep) cand[base + __popc(bal & ((1u << lane) - 1u))] = cb;
        __syncthreads();
        for (int c = 0; c < total; c++) {
            const int sb = cand[c];
            const int j = sb * B + t;
            if (j < P) stage[t] = sorted[j];
            __syncthreads();
            if (active && !(knn_point_box(q, blo[sb], bhi[sb]) > b2)) {
                const int n = min(B, P - sb * B);
                for (int k = 0; k < n; k++) knn_insert(knn_d(q, stage[k]), b0, b1, b2);
            }
            __syncthreads();
        }
    }
    if (active) dist2[__float_as_int(q.w)] = __fdiv_rn(__fadd_rn(__fadd_rn(b0, b1), b2), 3.f);
}
