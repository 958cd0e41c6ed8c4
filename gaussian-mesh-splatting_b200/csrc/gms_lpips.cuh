// gms_lpips.cuh -- LPIPS (VGG16, v0.1, forward only) as lpipsPyTorch computes it for metrics.py:74, sm_90a.
//
// The render and its ground truth run through VGG16 as one batch of two, NHWC activations [2,H,W,C]:
//   k_lpips_conv      conv3x3 (padding 1) + bias + ReLU as an implicit GEMM: rows = the 2*H*W pixels, columns = Cout,
//                     K = 9*Cin ordered (ky, kx, ci).  Tensor cores, mma.sync m16n8k8 TF32 with split operands
//                     (x = big + small, both TF32; big*big + big*small + small*big, FP32 accumulation): each product
//                     carries ~21 significant bits, so the conv is as accurate as an FP32 one (DESIGN.md 4.8).
//                     conv1_1 (K = 27, padded to 32) reads the two [3,H,W] images and applies the z-score in its loader,
//                     so the zero padding is zero in z-score space, as F.conv2d sees it.
//   k_lpips_pool      MaxPool2d(2, 2), floor.
//   k_lpips_head      per target map: per pixel f / (sqrt(sum_c f^2) + 1e-10) for both images, sum_c w[c] (fx - fy)^2,
//                     one double partial per block, pixels in a fixed order.
//   k_lpips_finalize  the partials of each layer in a fixed order, in double: term = sum / (H_l W_l); out = 5 terms, sum.
// No atomics: the same inputs give the same bits.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define GMS_LPIPS_BM 128         // GEMM rows (pixels) per block
#define GMS_LPIPS_BN 64          // GEMM columns (output channels) per block; every VGG16 Cout is a multiple
#define GMS_LPIPS_BK 16          // K per pipeline stage; every Cin but conv1_1's is a multiple, so a stage is one tap
#define GMS_LPIPS_LD 20          // shared row stride in floats: fragment reads (row g, column t) hit 32 distinct banks
#define GMS_LPIPS_STAGES 3
#define GMS_LPIPS_HEAD_PIX 256   // pixels per head block (8 warps x 32)

struct LpipsConv {
    const float* in;             // [2,H,W,Cin] (not conv1_1)
    const float* img;            // conv1_1: the two [3,H,W] images
    const float* gt;
    const float* w;              // [Cout][Kp]
    const float* bias;           // [Cout]
    float* out;                  // [2,H,W,Cout]
    int H, W, Cin, Cout, Kp;
};

__device__ __forceinline__ void lp_cp16(float* smem, const float* src, bool valid) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void lp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void lp_wait1() { asm volatile("cp.async.wait_group 1;\n" ::); }

// x = big + small exactly up to small's own TF32 rounding: x - big has at most 14 significant bits and is exact in FP32.
__device__ __forceinline__ void lp_split(float x, uint32_t& big, uint32_t& small) {
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(big) : "f"(x));
    const float r = __fsub_rn(x, __uint_as_float(big));
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(small) : "f"(r));
}

__device__ __forceinline__ void lp_mma(float* c, const uint32_t* a, const uint32_t* b) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// 128 threads, four warps as 2 x 2, each a 64 x 32 tile of the 128 x 64 block tile (4 x 4 mma tiles).
template <bool FIRST>
__global__ void __launch_bounds__(128) k_lpips_conv(LpipsConv p) {
    __shared__ __align__(16) float As[GMS_LPIPS_STAGES][GMS_LPIPS_BM][GMS_LPIPS_LD];
    __shared__ __align__(16) float Bs[GMS_LPIPS_STAGES][GMS_LPIPS_BN][GMS_LPIPS_LD];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
    const int H = p.H, W = p.W, HW = H * W, M = 2 * HW;
    const int m0 = blockIdx.x * GMS_LPIPS_BM, n0 = blockIdx.y * GMS_LPIPS_BN;
    const int nk = p.Kp / GMS_LPIPS_BK;
    const int q = tid & 3;      // 16-byte column of the cp.async loaders

    // the pixels this thread loads: rows (tid >> 2) + 32 i (conv1_1: row tid alone)
    int am[4], ay[4], ax[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int m = m0 + (FIRST ? tid : (tid >> 2) + 32 * i);
        const int pix = m < M ? (m < HW ? m : m - HW) : 0;
        am[i] = m; ay[i] = pix / W; ax[i] = pix - ay[i] * W;
    }

    auto load = [&](int s, int kc) {
        const int k0 = kc * GMS_LPIPS_BK;
        if (FIRST) {
            const bool row_ok = am[0] < M;
            const float* src = am[0] < HW ? p.img : p.gt;
#pragma unroll
            for (int j = 0; j < GMS_LPIPS_BK; j++) {
                const int k = k0 + j, tap = k / 3, ci = k - 3 * tap;
                const int yy = ay[0] + tap / 3 - 1, xx = ax[0] + tap % 3 - 1;
                float v = 0.f;
                if (row_ok && k < 27 && (unsigned)yy < (unsigned)H && (unsigned)xx < (unsigned)W) {
                    // lpipsPyTorch's z-score, (x - mean) / std with float32 buffers (-.030, -.088, -.188), (.458, .448, .450)
                    const float shift = ci == 0 ? -0.030f : ci == 1 ? -0.088f : -0.188f;
                    const float scale = ci == 0 ? 0.458f : ci == 1 ? 0.448f : 0.450f;
                    v = __fdiv_rn(__fsub_rn(src[(size_t)ci * HW + (size_t)yy * W + xx], shift), scale);
                }
                As[s][tid][j] = v;
            }
        } else {
            const int tap = k0 / p.Cin, c0 = k0 - tap * p.Cin + 4 * q, dy = tap / 3 - 1, dx = tap % 3 - 1;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int yy = ay[i] + dy, xx = ax[i] + dx;
                const bool ok = am[i] < M && (unsigned)yy < (unsigned)H && (unsigned)xx < (unsigned)W;
                const float* src = ok ? p.in + ((size_t)(am[i] + dy * W + dx) * p.Cin + c0) : p.in;
                lp_cp16(&As[s][(tid >> 2) + 32 * i][4 * q], src, ok);
            }
        }
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int n = (tid >> 2) + 32 * j;
            lp_cp16(&Bs[s][n][4 * q], p.w + (size_t)(n0 + n) * p.Kp + k0 + 4 * q, true);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
        for (int ni = 0; ni < 4; ni++)
#pragma unroll
            for (int r = 0; r < 4; r++) acc[mi][ni][r] = 0.f;

    for (int s = 0; s < GMS_LPIPS_STAGES - 1; s++) {
        if (s < nk) load(s, s);
        lp_commit();
    }
    for (int kc = 0; kc < nk; kc++) {
        lp_wait1();             // stage kc has landed (one younger group may still be in flight)
        __syncthreads();        // ... for every thread, and every warp is done with stage kc - 1, which the next load reuses
        if (kc + GMS_LPIPS_STAGES - 1 < nk) load((kc + GMS_LPIPS_STAGES - 1) % GMS_LPIPS_STAGES, kc + GMS_LPIPS_STAGES - 1);
        lp_commit();
        const int s = kc % GMS_LPIPS_STAGES;
#pragma unroll
        for (int kk = 0; kk < GMS_LPIPS_BK; kk += 8) {
            uint32_t ab[4][4], as[4][4], bb[4][2], bs[4][2];
#pragma unroll
            for (int mi = 0; mi < 4; mi++) {
                const int r = wm * 64 + mi * 16 + g;
                lp_split(As[s][r][kk + t], ab[mi][0], as[mi][0]);
                lp_split(As[s][r + 8][kk + t], ab[mi][1], as[mi][1]);
                lp_split(As[s][r][kk + t + 4], ab[mi][2], as[mi][2]);
                lp_split(As[s][r + 8][kk + t + 4], ab[mi][3], as[mi][3]);
            }
#pragma unroll
            for (int ni = 0; ni < 4; ni++) {
                const int c = wn * 32 + ni * 8 + g;
                lp_split(Bs[s][c][kk + t], bb[ni][0], bs[ni][0]);
                lp_split(Bs[s][c][kk + t + 4], bb[ni][1], bs[ni][1]);
            }
#pragma unroll
            for (int mi = 0; mi < 4; mi++)
#pragma unroll
                for (int ni = 0; ni < 4; ni++) {
                    lp_mma(acc[mi][ni], as[mi], bb[ni]);
                    lp_mma(acc[mi][ni], ab[mi], bs[ni]);
                    lp_mma(acc[mi][ni], ab[mi], bb[ni]);
                }
        }
    }

#pragma unroll
    for (int ni = 0; ni < 4; ni++) {
        const int n = n0 + wn * 32 + ni * 8 + 2 * t;
        const float b0 = p.bias[n], b1 = p.bias[n + 1];
#pragma unroll
        for (int mi = 0; mi < 4; mi++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int m = m0 + wm * 64 + mi * 16 + g + 8 * h;
                if (m < M)
                    *reinterpret_cast<float2*>(p.out + (size_t)m * p.Cout + n) =
                        make_float2(fmaxf(acc[mi][ni][2 * h] + b0, 0.f), fmaxf(acc[mi][ni][2 * h + 1] + b1, 0.f));
            }
    }
}

// [2,H,W,C] -> [2,H/2,W/2,C], one thread per output float4
__global__ void __launch_bounds__(256) k_lpips_pool(const float* __restrict__ in, int H, int W, int C, float* __restrict__ out) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)2 * Ho * Wo * C4) return;
    const int c4 = (int)(i % C4);
    size_t r = i / C4;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho), b = (int)(r / Ho);
    const float4* s = reinterpret_cast<const float4*>(in) + ((size_t)(b * H + 2 * yo) * W + 2 * xo) * C4 + c4;
    const float4 a = s[0], bq = s[C4], c = s[(size_t)W * C4], d = s[(size_t)(W + 1) * C4];
    reinterpret_cast<float4*>(out)[i] = make_float4(fmaxf(fmaxf(a.x, bq.x), fmaxf(c.x, d.x)), fmaxf(fmaxf(a.y, bq.y), fmaxf(c.y, d.y)),
                                                    fmaxf(fmaxf(a.z, bq.z), fmaxf(c.z, d.z)), fmaxf(fmaxf(a.w, bq.w), fmaxf(c.w, d.w)));
}

__device__ __forceinline__ float lp_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// NC = C / 32 channels per lane.  One warp per pixel, 32 consecutive pixels per warp, 8 warps per block.
template <int NC>
__global__ void __launch_bounds__(256) k_lpips_head(const float* __restrict__ f, int HW, const float* __restrict__ lin,
                                                    double* __restrict__ part) {
    __shared__ double ws[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[NC];
#pragma unroll
    for (int j = 0; j < NC; j++) w[j] = lin[lane + 32 * j];
    double acc = 0.0;
    const int p0 = blockIdx.x * GMS_LPIPS_HEAD_PIX + warp * 32;
    for (int k = 0; k < 32 && p0 + k < HW; k++) {
        const float* fx = f + (size_t)(p0 + k) * (NC * 32);
        const float* fy = fx + (size_t)HW * (NC * 32);
        float x[NC], y[NC], sx = 0.f, sy = 0.f;
#pragma unroll
        for (int j = 0; j < NC; j++) {
            x[j] = fx[lane + 32 * j]; y[j] = fy[lane + 32 * j];
            sx = fmaf(x[j], x[j], sx); sy = fmaf(y[j], y[j], sy);
        }
        const float nx = sqrtf(lp_warp_sum(sx)) + 1e-10f, ny = sqrtf(lp_warp_sum(sy)) + 1e-10f;
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < NC; j++) {
            const float d = x[j] / nx - y[j] / ny;
            s = fmaf(w[j], d * d, s);
        }
        acc += (double)lp_warp_sum(s);
    }
    if (lane == 0) ws[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0;
        for (int i = 0; i < 8; i++) a += ws[i];
        part[blockIdx.x] = a;
    }
}

struct LpipsFinal {
    const double* part[5];
    int blocks[5];
    double inv_hw[5];
};

// one block of 256: per layer, strided sums in a fixed order, then a fixed tree
__global__ void __launch_bounds__(256) k_lpips_finalize(LpipsFinal f, float* __restrict__ out) {
    __shared__ double s[256];
    double total = 0.0;
    for (int l = 0; l < 5; l++) {
        double a = 0.0;
        for (int i = threadIdx.x; i < f.blocks[l]; i += 256) a += f.part[l][i];
        s[threadIdx.x] = a;
        __syncthreads();
        for (int w = 128; w > 0; w >>= 1) {
            if ((int)threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            const float term = (float)(s[0] * f.inv_hw[l]);
            out[l] = term;
            total += (double)term;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) out[5] = (float)total;
}
