// gms_image.cuh -- image sink / source kernels: float CHW <-> 8-bit interleaved rows, sm_90a.
//
// Sink: replaces the device half of torchvision.utils.save_image as the reference's render scripts call it
// (scripts/render_time_animated.py:86-87, scripts/render.py): make_grid is the identity for one image, then
// `img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8)` -- four full-size ATen passes and a
// strided 24.9 MB fp32 device->host copy per 1080p frame.  Here one kernel quantises and interleaves into the exact byte
// layout the encoder consumes (optionally with PNG's per-row filter byte), so the copy is 6.2 MB of uint8 and the host
// only deflates.  Source: the inverse (uint8 HWC or CHW -> float CHW / 255, torchvision ToTensor semantics,
// utils/general_utils.py PILtoTorch:105-112) for ground-truth images kept as 8-bit data.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// save_image's byte: mul(255).add(0.5).clamp(0, 255).to(uint8) -- two roundings (mul, add) like ATen's separate passes, then
// truncation.  NaN -> 0 (fmaxf returns the non-NaN operand).  Shared with the metric kernel's 8-bit round trip.
__device__ __forceinline__ uint8_t gms_quantize_u8(float x) {
    const float v = __fadd_rn(__fmul_rn(x, 255.0f), 0.5f);
    return (uint8_t)fminf(fmaxf(v, 0.0f), 255.0f);
}
// ToTensor: byte / 255
__device__ __forceinline__ float gms_dequantize_u8(uint8_t b) { return __fdiv_rn((float)b, 255.0f); }

// one thread per pixel: reads C coalesced planes, writes C adjacent bytes.  row_prefix: bytes reserved at the start of
// every output row (1 for PNG: the filter-type byte, written as 0 = "None").
__global__ void __launch_bounds__(256)
k_image_quantize(const float* __restrict__ chw, uint8_t* __restrict__ out, int C, int H, int W, int row_prefix) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t HW = (size_t)H * W, pix = (size_t)y * W + x;
    uint8_t* row = out + (size_t)y * ((size_t)W * C + row_prefix);
    if (row_prefix && x == 0)
        for (int k = 0; k < row_prefix; k++) row[k] = 0;
    uint8_t* px = row + row_prefix + (size_t)x * C;
    for (int c = 0; c < C; c++) px[c] = gms_quantize_u8(chw[c * HW + pix]);
}

__global__ void __launch_bounds__(256)
k_image_dequantize(const uint8_t* __restrict__ src, int src_is_hwc, float* __restrict__ chw, int C, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t HW = (size_t)H * W, pix = (size_t)y * W + x;
    for (int c = 0; c < C; c++) {
        const uint8_t b = src_is_hwc ? src[pix * C + c] : src[c * HW + pix];
        chw[c * HW + pix] = gms_dequantize_u8(b);
    }
}
