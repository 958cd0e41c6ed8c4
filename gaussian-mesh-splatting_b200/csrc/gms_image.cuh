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

// The remote viewer's byte (train.py:72-74): `(torch.clamp(img, 0, 1) * 255).byte()` as ATen computes it on the device.
// clamp keeps NaN (ATen's clamp kernel returns a NaN input as is), one rounded multiply, then c10's float -> uint8 cast,
// which goes through int64: the conversion truncates toward zero and turns NaN into 0.  Unlike gms_quantize_u8 nothing is
// rounded, so 0.999 gives 254, not 255.
__device__ __forceinline__ uint8_t gms_clamp_u8(float x) {
    const float c = isnan(x) ? x : fminf(fmaxf(x, 0.0f), 1.0f);
    return (uint8_t)(long long)__fmul_rn(c, 255.0f);
}

// one thread per pixel: reads C coalesced planes, writes the pixel's C bytes of the packed [H,W,C] image
__global__ void __launch_bounds__(256)
k_image_clamp_u8(const float* __restrict__ chw, uint8_t* __restrict__ hwc, int C, int H, int W) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const size_t HW = (size_t)H * W, pix = (size_t)y * W + x;
    uint8_t* px = hwc + pix * C;
    for (int c = 0; c < C; c++) px[c] = gms_clamp_u8(chw[c * HW + pix]);
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

// ---- ground-truth preparation of the dataset loader (gms_b200/dataset.py) -----------------------------------------------

// readCamerasFromTransforms' RGBA -> RGB (scene/dataset_readers.py:204-210), the numpy sequence in float64 step by step:
//   n = u / 255.0;  arr = n_rgb * n_a + bg * (1 - n_a);  byte = (int)(arr * 255.0)
// Every operation is an explicit round-to-nearest intrinsic so nvcc cannot contract a multiply-add into an FMA (the result
// would differ from numpy in ~150 of the 65,536 (value, alpha) pairs per background).  arr * 255.0 lies in [0, 255], so
// the truncating conversion is numpy's float -> int8 cast read back as a byte.
__device__ __forceinline__ uint8_t gms_composite_u8(uint8_t v, double a, double bg_term) {
    const double n = __ddiv_rn((double)v, 255.0);
    return (uint8_t)(int)__dmul_rn(__dadd_rn(__dmul_rn(n, a), bg_term), 255.0);
}

// one thread per pixel: 4 bytes in, 3 bytes out
__global__ void __launch_bounds__(256)
k_image_composite_rgba(const uchar4* __restrict__ rgba, uint8_t* __restrict__ rgb, long long npix, double bg) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const uchar4 p = rgba[i];
    const double a = __ddiv_rn((double)p.w, 255.0);
    const double bg_term = __dmul_rn(bg, __dsub_rn(1.0, a));
    uint8_t* o = rgb + 3 * i;
    o[0] = gms_composite_u8(p.x, a, bg_term);
    o[1] = gms_composite_u8(p.y, a, bg_term);
    o[2] = gms_composite_u8(p.z, a, bg_term);
}

// Pillow's ImagingResample, 8-bit path (libImaging/Resample.c ResampleHorizontal_8bpc / ResampleVertical_8bpc), for
// 3-channel interleaved rows.  The host builds each axis' table (gms_b200/dataset.py resize_coeffs): per output index i,
// bounds[2i] = first source index, bounds[2i+1] = tap count n, and coeffs[i*ksize + t] the 22-bit fixed-point weight of tap t.
// Each output byte is clamp(((1 << 21) + sum_t src[bounds+t] * k[t]) >> 22, 0, 255), summed in int32 in tap order.
#define GMS_RESAMPLE_BITS 22

__device__ __forceinline__ uint8_t gms_resample_clip8(int ss) {
    const int v = ss >> GMS_RESAMPLE_BITS;      // arithmetic shift, as Pillow's clip8
    return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: output row y reads source row row0 + y.  One thread per output pixel.
__global__ void __launch_bounds__(256)
k_resize_h_u8(const uint8_t* __restrict__ src, int in_w, uint8_t* __restrict__ dst, int out_w, int row0,
              const int* __restrict__ bounds, const int* __restrict__ coeffs, int ksize) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= out_w) return;
    const int xmin = bounds[2 * x], n = bounds[2 * x + 1];
    const int* k = coeffs + (size_t)x * ksize;
    const uint8_t* s = src + ((size_t)(row0 + y) * in_w + xmin) * 3;
    int s0 = 1 << (GMS_RESAMPLE_BITS - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < n; t++) {
        const int w = k[t];
        s0 += s[3 * t + 0] * w;
        s1 += s[3 * t + 1] * w;
        s2 += s[3 * t + 2] * w;
    }
    uint8_t* o = dst + ((size_t)y * out_w + x) * 3;
    o[0] = gms_resample_clip8(s0);
    o[1] = gms_resample_clip8(s1);
    o[2] = gms_resample_clip8(s2);
}

// vertical pass: output row y reads source rows bounds[2y] - row0 ...  One thread per output pixel; neighbouring threads read
// neighbouring bytes of the same source rows.
__global__ void __launch_bounds__(256)
k_resize_v_u8(const uint8_t* __restrict__ src, int w, uint8_t* __restrict__ dst, int row0,
              const int* __restrict__ bounds, const int* __restrict__ coeffs, int ksize) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const int ymin = bounds[2 * y] - row0, n = bounds[2 * y + 1];
    const int* k = coeffs + (size_t)y * ksize;
    const size_t stride = (size_t)w * 3;
    const uint8_t* s = src + (size_t)ymin * stride + (size_t)x * 3;
    int s0 = 1 << (GMS_RESAMPLE_BITS - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < n; t++) {
        const int wt = k[t];
        const uint8_t* r = s + t * stride;
        s0 += r[0] * wt;
        s1 += r[1] * wt;
        s2 += r[2] * wt;
    }
    uint8_t* o = dst + ((size_t)y * w + x) * 3;
    o[0] = gms_resample_clip8(s0);
    o[1] = gms_resample_clip8(s1);
    o[2] = gms_resample_clip8(s2);
}
