// gms_anomaly.cuh -- the NaN scan of anomaly detection (gms_nan_scan, the training frames' anomaly hooks).
//
// A pure streaming read: every float of the scanned buffers is loaded once (128-bit loads over the 16-byte-aligned body,
// scalar loads for the head before it and the tail after it), each thread keeps the smallest index it saw, one block-level
// reduction finds the block's smallest, and only a block that saw a NaN makes its one atomicMin on the record.  A clean
// scan writes nothing.
#pragma once
#include <stdint.h>

#define GMS_NAN_BLOCK 256
#define GMS_NAN_UNROLL 4        // independent 128-bit loads in flight per thread

struct GmsNanBuf {
    const float* ptr;
    int64_t n;
    int64_t head;       // scalar elements before the first 16-byte boundary (<= 3, <= n)
    uint64_t key;       // stage << 56 | tensor << 48
};
struct GmsNanTable { GmsNanBuf b[GMS_NAN_SCAN_MAX_BUFFERS]; };

// NaN by its bits (exponent all ones, mantissa non-zero): independent of any fast-math treatment of comparisons.
__device__ __forceinline__ bool gms_is_nan(float x) { return (__float_as_uint(x) & 0x7fffffffu) > 0x7f800000u; }

// Index (0..3) of the first NaN lane of v, or 4.
__device__ __forceinline__ int gms_first_nan4(float4 v) {
    return gms_is_nan(v.x) ? 0 : gms_is_nan(v.y) ? 1 : gms_is_nan(v.z) ? 2 : gms_is_nan(v.w) ? 3 : 4;
}

// blockIdx.y = buffer; blockIdx.x strides over the buffer's float4 body.  Block x == 0 also reads the head and the tail.
__global__ void __launch_bounds__(GMS_NAN_BLOCK) k_nan_scan(GmsNanTable t, uint64_t* record) {
    const GmsNanBuf b = t.b[blockIdx.y];
    const int64_t n4 = (b.n - b.head) >> 2;
    const float4* body = reinterpret_cast<const float4*>(b.ptr + b.head);
    const int64_t stride = (int64_t)gridDim.x * GMS_NAN_BLOCK;
    uint64_t first = ~0ull;
    int64_t j = (int64_t)blockIdx.x * GMS_NAN_BLOCK + threadIdx.x;
    // a thread visits its elements in increasing order: its first NaN is its smallest index
    for (; j + (GMS_NAN_UNROLL - 1) * stride < n4 && first == ~0ull; j += GMS_NAN_UNROLL * stride) {
        float4 v[GMS_NAN_UNROLL];
#pragma unroll
        for (int u = 0; u < GMS_NAN_UNROLL; u++) v[u] = __ldcs(body + j + u * stride);
#pragma unroll
        for (int u = GMS_NAN_UNROLL - 1; u >= 0; u--) {
            const int c = gms_first_nan4(v[u]);
            if (c < 4) first = (uint64_t)(b.head + 4 * (j + u * stride) + c);
        }
    }
    for (; j < n4 && first == ~0ull; j += stride) {
        const int c = gms_first_nan4(__ldcs(body + j));
        if (c < 4) first = (uint64_t)(b.head + 4 * j + c);
    }
    if (blockIdx.x == 0 && threadIdx.x < 8) {
        const int64_t tail0 = b.head + 4 * n4;
        const int64_t i = threadIdx.x < 4 ? (int64_t)threadIdx.x : tail0 + (threadIdx.x - 4);
        const bool in = threadIdx.x < 4 ? i < b.head : i < b.n;
        if (in && gms_is_nan(b.ptr[i]) && (uint64_t)i < first) first = (uint64_t)i;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const uint64_t other = __shfl_xor_sync(0xffffffffu, first, o);
        first = other < first ? other : first;
    }
    __shared__ uint64_t s_min[GMS_NAN_BLOCK / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) s_min[warp] = first;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t m = s_min[0];
#pragma unroll
        for (int w = 1; w < GMS_NAN_BLOCK / 32; w++) m = s_min[w] < m ? s_min[w] : m;
        if (m != ~0ull) atomicMin(reinterpret_cast<unsigned long long*>(record), (unsigned long long)(b.key | m));
    }
}
