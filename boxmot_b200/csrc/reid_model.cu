// reid_model.cu -- ReID appearance-embedding path on the GPU: detection crops -> OSNet -> L2-normalised rows.
//
// Replaces (relative to /root/reference/boxmot):
//   reid/backends/base_backend.py:148-207   get_crops (cv2.resize INTER_LINEAR, BGR2RGB, /255, mean/std) and
//                                           get_features (forward + row-wise L2 normalisation)
//   reid/backbones/osnet.py:27-260,380-405  ConvLayer / Conv1x1 / Conv1x1Linear / LightConv3x3 / ChannelGate /
//                                           OSBlock / OSNet.forward (eval mode, BatchNorm folded offline)
//   native/cpp/trackers/base/src/reid_onnx.cpp:51-383  (per-crop batch-1 ORT forward of the native path)
//
// Data layout: activations are NHWC float32 in HBM, one chunk of crops at a time (256 by default: one
// full-width chunk keeps the small, latency-bound tile kernels in full waves); weights are a BN-folded float32 blob
// (boxmot_b200/weights.py) uploaded once.  Round-1 kernels are float32 CUDA-core kernels with shared-memory
// tiling; every 1x1 convolution goes through one GEMM-shaped kernel (k_pointwise) whose prologue can build
// the gated branch sum on the fly and whose epilogue fuses bias / residual / ReLU.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <algorithm>
#include <fstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "engine.h"
#include "pointwise_tc.cuh"
#include "cspreid_kernels.cuh"
#include "hacnn_kernels.cuh"
#include "mlfn_kernels.cuh"
#include "resnet_tc.cuh"
#include "vit_tc.cuh"

namespace bmb {

#define RCUDA_OK(expr)                                                                                  \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess)                                                                          \
            throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e));              \
    } while (0)

constexpr int IN_H = 256, IN_W = 128;
constexpr int IN_H_MAX = 384;   // LMBN_n crops are 384x128
constexpr int IN_W_MAX = 256;   // CLIP vehicle crops are 256x256 (every other model's width is 128)
constexpr uint32_t BLOB_MAGIC = 0x45523242u;

// streaming multiprocessors of the current device: grid-stride kernels launch a few CTAs per SM
static int sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 0;
    return n > 0 ? n : 132;
}

__device__ __forceinline__ int chunk_count(const int* d_n, int off, int cap) {
    int n = *d_n - off;
    n = n < 0 ? 0 : n;
    return n > cap ? cap : n;
}

// ---------------------------------------------------------------------------------------------------
// K1: crop + OpenCV-exact bilinear resize + BGR->RGB + /255 + mean/std  ->  (N,in_h,in_w,3) float32
// One CTA per crop.  cv2.resize(INTER_LINEAR) on uint8 is integer arithmetic: 11-bit coefficients derived from a
// float32 phase, horizontal pass in int32, vertical (((b0*(S0>>4))>>16)+((b1*(S1>>4))>>16)+2)>>2.  x phases are
// clamped at the borders, y rows are clipped at fetch (pinned against cv2 in tests/test_oracle_reid.py).
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void linear_coeff(int d, int src_n, double scale, bool clamp, int& idx, int& a0, int& a1) {
    float f = (float)(((double)d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f = f - (float)s;
    if (clamp) {
        if (s < 0) { s = 0; f = 0.f; }
        if (s >= src_n - 1) { s = src_n - 1; f = 0.f; }
    }
    idx = s;
    a0 = (int)rintf((1.0f - f) * 2048.0f);
    a1 = (int)rintf(f * 2048.0f);
}

// per-channel (RGB) mean and std of the staged crop: ImageNet's for every model but CLIP (0.5, base_backend.py:52-54)
struct CropNorm { float mean[3], std[3]; };
constexpr CropNorm kImageNetNorm{{0.485f, 0.456f, 0.406f}, {0.229f, 0.224f, 0.225f}};

__global__ void __launch_bounds__(256) k_crop_resize_norm(const uint8_t* __restrict__ images, size_t image_stride,
                                                          int rows, int cols, const CropDesc* __restrict__ crops,
                                                          const int* __restrict__ d_n, int off, int cap,
                                                          float* __restrict__ blob, int pad_mode, int in_h, int in_w,
                                                          CropNorm nm) {
    const int n = blockIdx.x;
    if (n >= chunk_count(d_n, off, cap)) return;
    const CropDesc cd = crops[off + n];
    __shared__ int xi[IN_W_MAX], xa0[IN_W_MAX], xa1[IN_W_MAX];
    __shared__ int yi[IN_H_MAX], ya0[IN_H_MAX], ya1[IN_H_MAX];
    // box.round().astype(int): round half to even
    const int x1 = (int)rintf(cd.x1), y1 = (int)rintf(cd.y1), x2 = (int)rintf(cd.x2), y2 = (int)rintf(cd.y2);
    const int cx1 = max(0, x1), cy1 = max(0, y1), cx2 = min(cols, x2), cy2 = min(rows, y2);
    const bool valid = cx2 > cx1 && cy2 > cy1;
    const int sw = cx2 - cx1, sh = cy2 - cy1;
    // resize_pad (preprocessing.py:21-45): scale = min(W / w, H / h); new = int(size * scale); centred, ImageNet-mean border
    int nw = in_w, nh = in_h, pl = 0, pt = 0;
    if (valid && pad_mode) {
        const double sc = fmin((double)in_w / (double)sw, (double)in_h / (double)sh);
        nw = max(1, (int)((double)sw * sc));
        nh = max(1, (int)((double)sh * sc));
        pl = (in_w - nw) / 2;
        pt = (in_h - nh) / 2;
    }
    if (valid) {
        const double sx = 1.0 / ((double)nw / (double)sw), sy = 1.0 / ((double)nh / (double)sh);
        for (int d = threadIdx.x; d < nw; d += blockDim.x) linear_coeff(d, sw, sx, true, xi[d], xa0[d], xa1[d]);
        for (int d = threadIdx.x; d < nh; d += blockDim.x) linear_coeff(d, sh, sy, false, yi[d], ya0[d], ya1[d]);
    }
    __syncthreads();
    const uint8_t* img = images + (size_t)cd.image * image_stride;
    float* out = blob + (size_t)n * in_h * in_w * 3;
    for (int p = threadIdx.x; p < in_h * in_w; p += blockDim.x) {
        const int py = p / in_w, px = p - py * in_w;
        const int dy = py - pt, dx = px - pl;
        int v[3] = {0, 0, 0};
        if (valid && (dx < 0 || dx >= nw || dy < 0 || dy >= nh)) {
            v[0] = 104; v[1] = 116; v[2] = 124;      // IMAGENET_MEAN_BGR (the crop is BGR until the channel flip below)
        } else if (valid) {
            const int sx0 = xi[dx], sx1 = min(sx0 + 1, sw - 1);
            const int r0 = min(max(yi[dy], 0), sh - 1), r1 = min(max(yi[dy] + 1, 0), sh - 1);
            const uint8_t* p0 = img + ((size_t)(cy1 + r0) * cols + cx1) * 3;
            const uint8_t* p1 = img + ((size_t)(cy1 + r1) * cols + cx1) * 3;
            const int a0 = xa0[dx], a1 = xa1[dx], b0 = ya0[dy], b1 = ya1[dy];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int h0 = (int)p0[sx0 * 3 + c] * a0 + (int)p0[sx1 * 3 + c] * a1;
                const int h1 = (int)p1[sx0 * 3 + c] * a0 + (int)p1[sx1 * 3 + c] * a1;
                int r = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
                v[c] = min(max(r, 0), 255);
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {  // output channel c is RGB: source channel 2-c
            const float f = __fdiv_rn((float)v[2 - c], 255.0f);
            out[(size_t)p * 3 + c] = __fdiv_rn(f - nm.mean[c], nm.std[c]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// K2: stem 7x7 stride-2 conv (3 -> C0) + folded BN + ReLU : (N,in_h,128,3) -> (N,in_h/2,64,C0)
// CTA = 8 output rows x 64 columns of one crop; the 21 x 134 x 3 input window and the weight chunk live in
// shared memory; a thread owns two output pixels (x, x+32) x 16 output channels.
// ---------------------------------------------------------------------------------------------------
// RAW (the instance-norm stem of OSNet-AIN / OSNet-IBN): no bias, no ReLU; the instance norm and the ReLU are applied by
// k_maxpool3s2_in.
constexpr int ST_R = 8, ST_IR = 2 * ST_R + 5, ST_IC = IN_W + 6;
template <bool RAW = false>
__global__ void __launch_bounds__(256) k_stem(const float* __restrict__ blob, const float* __restrict__ w,
                                              const float* __restrict__ bias, int C0, const int* __restrict__ d_n,
                                              int off, int cap, float* __restrict__ out, int in_h) {
    const int n = blockIdx.y;
    if (n >= chunk_count(d_n, off, cap)) return;
    extern __shared__ __align__(16) float smem[];
    float* sin = smem;                         // [ST_IR][ST_IC][3]
    float* sw = smem + ((ST_IR * ST_IC * 3 + 3) & ~3);  // [147][16], 16-byte aligned for float4 reads
    const int oy0 = blockIdx.x * ST_R;
    const int iy0 = oy0 * 2 - 3;
    const float* src = blob + (size_t)n * in_h * IN_W * 3;
    for (int e = threadIdx.x; e < ST_IR * ST_IC * 3; e += blockDim.x) {
        const int r = e / (ST_IC * 3), rem = e - r * (ST_IC * 3);
        const int cidx = rem / 3, ch = rem - cidx * 3;
        const int iy = iy0 + r, ix = cidx - 3;
        sin[e] = (iy >= 0 && iy < in_h && ix >= 0 && ix < IN_W) ? src[((size_t)iy * IN_W + ix) * 3 + ch] : 0.f;
    }
    const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
    for (int co0 = 0; co0 < C0; co0 += 16) {
        __syncthreads();
        for (int e = threadIdx.x; e < 147 * 16; e += blockDim.x) {
            const int k = e >> 4, c = e & 15;
            sw[e] = w[(size_t)k * C0 + co0 + c];
        }
        __syncthreads();
        // two output channels per float2, IEEE fmaf per lane
        float2 acc0[8], acc1[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) { acc0[c] = make_float2(0.f, 0.f); acc1[c] = make_float2(0.f, 0.f); }
        for (int kh = 0; kh < 7; ++kh) {
            const float* row = sin + (size_t)(ty * 2 + kh) * ST_IC * 3;
            for (int kw = 0; kw < 7; ++kw) {
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const float a0 = row[(tx * 2 + kw) * 3 + ci];
                    const float a1 = row[((tx + 32) * 2 + kw) * 3 + ci];
                    const float2 a0p = make_float2(a0, a0), a1p = make_float2(a1, a1);
                    const float4* wp = reinterpret_cast<const float4*>(sw + ((kh * 7 + kw) * 3 + ci) * 16);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float4 wv = wp[q];
                        const float2 w01 = make_float2(wv.x, wv.y), w23 = make_float2(wv.z, wv.w);
                        acc0[q * 2 + 0] = um::ffma2(a0p, w01, acc0[q * 2 + 0]);
                        acc0[q * 2 + 1] = um::ffma2(a0p, w23, acc0[q * 2 + 1]);
                        acc1[q * 2 + 0] = um::ffma2(a1p, w01, acc1[q * 2 + 0]);
                        acc1[q * 2 + 1] = um::ffma2(a1p, w23, acc1[q * 2 + 1]);
                    }
                }
            }
        }
        float* o0 = out + (((size_t)n * (in_h / 2) + oy0 + ty) * 64 + tx) * C0 + co0;
        float* o1 = o0 + (size_t)32 * C0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (RAW) {
                reinterpret_cast<float4*>(o0)[q] = make_float4(acc0[q * 2].x, acc0[q * 2].y, acc0[q * 2 + 1].x, acc0[q * 2 + 1].y);
                reinterpret_cast<float4*>(o1)[q] = make_float4(acc1[q * 2].x, acc1[q * 2].y, acc1[q * 2 + 1].x, acc1[q * 2 + 1].y);
                continue;
            }
            const float4 b = *reinterpret_cast<const float4*>(bias + co0 + q * 4);
            float4 r0 = make_float4(fmaxf(acc0[q * 2].x + b.x, 0.f), fmaxf(acc0[q * 2].y + b.y, 0.f),
                                    fmaxf(acc0[q * 2 + 1].x + b.z, 0.f), fmaxf(acc0[q * 2 + 1].y + b.w, 0.f));
            float4 r1 = make_float4(fmaxf(acc1[q * 2].x + b.x, 0.f), fmaxf(acc1[q * 2].y + b.y, 0.f),
                                    fmaxf(acc1[q * 2 + 1].x + b.z, 0.f), fmaxf(acc1[q * 2 + 1].y + b.w, 0.f));
            reinterpret_cast<float4*>(o0)[q] = r0;
            reinterpret_cast<float4*>(o1)[q] = r1;
        }
    }
}

// K3: max pool 3x3 stride 2 pad 1 : (N,H,W,C) -> (N,H/2,W/2,C)
__global__ void k_maxpool3s2(const float* __restrict__ in, int H, int W, int C, const int* __restrict__ d_n, int off,
                             int cap, float* __restrict__ out) {
    const int n_crops = chunk_count(d_n, off, cap);
    const int OH = H / 2, OW = W / 2, C4 = C / 4;
    const size_t total = (size_t)n_crops * OH * OW * C4;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(e % C4);
        size_t r = e / C4;
        const int ox = (int)(r % OW); r /= OW;
        const int oy = (int)(r % OH);
        const int n = (int)(r / OH);
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * 2 - 1 + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * 2 - 1 + kx;
                if (ix < 0 || ix >= W) continue;
                const float4 v = *reinterpret_cast<const float4*>(in + (((size_t)n * H + iy) * W + ix) * C + c4 * 4);
                m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
            }
        }
        *reinterpret_cast<float4*>(out + (((size_t)n * OH + oy) * OW + ox) * C + c4 * 4) = m;
    }
}

// K4: average pool 2x2 stride 2
__global__ void k_avgpool2(const float* __restrict__ in, int H, int W, int C, const int* __restrict__ d_n, int off,
                           int cap, float* __restrict__ out) {
    const int n_crops = chunk_count(d_n, off, cap);
    const int OH = H / 2, OW = W / 2, C4 = C / 4;
    const size_t total = (size_t)n_crops * OH * OW * C4;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(e % C4);
        size_t r = e / C4;
        const int ox = (int)(r % OW); r /= OW;
        const int oy = (int)(r % OH);
        const int n = (int)(r / OH);
        const float* p = in + (((size_t)n * H + oy * 2) * W + ox * 2) * C + c4 * 4;
        const float4 a = *reinterpret_cast<const float4*>(p);
        const float4 b = *reinterpret_cast<const float4*>(p + C);
        const float4 c = *reinterpret_cast<const float4*>(p + (size_t)W * C);
        const float4 d = *reinterpret_cast<const float4*>(p + (size_t)W * C + C);
        float4 o;
        o.x = (a.x + b.x + c.x + d.x) * 0.25f; o.y = (a.y + b.y + c.y + d.y) * 0.25f;
        o.z = (a.z + b.z + c.z + d.z) * 0.25f; o.w = (a.w + b.w + c.w + d.w) * 0.25f;
        *reinterpret_cast<float4*>(out + (((size_t)n * OH + oy) * OW + ox) * C + c4 * 4) = o;
    }
}

// ---------------------------------------------------------------------------------------------------
// K4b: InstanceNorm2d(affine=True, track_running_stats=False) of OSNet-AIN / OSNet-IBN on NHWC maps [crops][HW][C]:
//   y = (x - mean_nc) / sqrt(var_nc + 1e-5) * gamma_c + beta_c,  mean / biased var over the crop's H x W.
// Statistics: one CTA per (32-channel group, crop); lane = channel, eight pixel stripes of four float64 partial sums
// each, combined in a fixed order, so a crop's statistics do not depend on the chunk it lands in or its position in it.
// No floating-point atomics.  Output per (crop, channel): {mean, 1 / sqrt(var + eps)} in float64.
// Apply: (x - mean) is taken in float64 and rounded once, then scaled by gamma * rstd and shifted by beta in float32
// (no cancellation between x * scale and mean * scale when a channel is nearly constant).
// ---------------------------------------------------------------------------------------------------
constexpr int INS_LANES = 32, INS_STRIPES = 8;
__global__ void __launch_bounds__(INS_LANES * INS_STRIPES) k_in_stats(const float* __restrict__ x, int HW, int C,
                                                                      const int* __restrict__ d_n, int off, int cap,
                                                                      double2* __restrict__ stats) {
    const int n = blockIdx.y;
    if (n >= chunk_count(d_n, off, cap)) return;
    const int lane = threadIdx.x % INS_LANES, g = threadIdx.x / INS_LANES;
    const int c = blockIdx.x * INS_LANES + lane;
    __shared__ double s_sum[INS_STRIPES][INS_LANES], s_sq[INS_STRIPES][INS_LANES];
    double s[4] = {0.0, 0.0, 0.0, 0.0}, q[4] = {0.0, 0.0, 0.0, 0.0};
    if (c < C) {
        const float* xp = x + (size_t)n * HW * C + c;
        int p = g;
        for (; p + 3 * INS_STRIPES < HW; p += 4 * INS_STRIPES) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const double v = (double)__ldg(xp + (size_t)(p + u * INS_STRIPES) * C);
                s[u] += v;
                q[u] = fma(v, v, q[u]);
            }
        }
        for (; p < HW; p += INS_STRIPES) {
            const double v = (double)__ldg(xp + (size_t)p * C);
            s[0] += v;
            q[0] = fma(v, v, q[0]);
        }
    }
    s_sum[g][lane] = (s[0] + s[1]) + (s[2] + s[3]);
    s_sq[g][lane] = (q[0] + q[1]) + (q[2] + q[3]);
    __syncthreads();
    if (g == 0 && c < C) {
        double ts = 0.0, tq = 0.0;
        for (int k = 0; k < INS_STRIPES; ++k) { ts += s_sum[k][lane]; tq += s_sq[k][lane]; }
        const double mean = ts / (double)HW;
        const double var = fmax(tq / (double)HW - mean * mean, 0.0);
        stats[(size_t)n * C + c] = make_double2(mean, 1.0 / sqrt(var + 1e-5));
    }
}

__device__ __forceinline__ float in_apply1(float x, double2 st, float gamma, float beta) {
    return fmaf((float)((double)x - st.x), (float)(st.y * (double)gamma), beta);
}

// out = act(IN(x) * gamma + beta (+ residual)); out may alias x or residual (element-wise, each element read once
// before it is written).  act: 0 none, 1 ReLU.
__global__ void k_in_apply(const float* x, const float* residual, float* out, int HW, int C,
                           const float* __restrict__ gamma, const float* __restrict__ beta,
                           const double2* __restrict__ stats, int relu, const int* __restrict__ d_n, int off, int cap) {
    const int n_crops = chunk_count(d_n, off, cap);
    const int C4 = C / 4;
    const size_t per_crop = (size_t)HW * C4, total = (size_t)n_crops * per_crop;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(e % C4) * 4;
        const size_t n = e / per_crop;
        const double2* st = stats + n * C + c;
        const float4 v = reinterpret_cast<const float4*>(x)[e];
        const float4 gm = *reinterpret_cast<const float4*>(gamma + c);
        const float4 bt = *reinterpret_cast<const float4*>(beta + c);
        float4 y = make_float4(in_apply1(v.x, st[0], gm.x, bt.x), in_apply1(v.y, st[1], gm.y, bt.y),
                               in_apply1(v.z, st[2], gm.z, bt.z), in_apply1(v.w, st[3], gm.w, bt.w));
        if (residual) {
            const float4 r = reinterpret_cast<const float4*>(residual)[e];
            y.x += r.x; y.y += r.y; y.z += r.z; y.w += r.w;
        }
        if (relu) { y.x = fmaxf(y.x, 0.f); y.y = fmaxf(y.y, 0.f); y.z = fmaxf(y.z, 0.f); y.w = fmaxf(y.w, 0.f); }
        reinterpret_cast<float4*>(out)[e] = y;
    }
}

// K3 with the instance-norm stem fused in: max over the 3x3 window of relu(IN(x) * gamma + beta), applied per element
// before the max (gamma may be negative, so the norm does not commute with the max).
__global__ void k_maxpool3s2_in(const float* __restrict__ in, int H, int W, int C, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const double2* __restrict__ stats,
                                const int* __restrict__ d_n, int off, int cap, float* __restrict__ out) {
    const int n_crops = chunk_count(d_n, off, cap);
    const int OH = H / 2, OW = W / 2, C4 = C / 4;
    const size_t total = (size_t)n_crops * OH * OW * C4;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(e % C4);
        size_t r = e / C4;
        const int ox = (int)(r % OW); r /= OW;
        const int oy = (int)(r % OH);
        const int n = (int)(r / OH);
        const double2* st = stats + (size_t)n * C + c4 * 4;
        const double2 s0 = st[0], s1 = st[1], s2 = st[2], s3 = st[3];
        const float4 gm = *reinterpret_cast<const float4*>(gamma + c4 * 4);
        const float4 bt = *reinterpret_cast<const float4*>(beta + c4 * 4);
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f);   // every window holds a valid pixel and ReLU output is >= 0
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * 2 - 1 + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * 2 - 1 + kx;
                if (ix < 0 || ix >= W) continue;
                const float4 v = *reinterpret_cast<const float4*>(in + (((size_t)n * H + iy) * W + ix) * C + c4 * 4);
                m.x = fmaxf(m.x, in_apply1(v.x, s0, gm.x, bt.x)); m.y = fmaxf(m.y, in_apply1(v.y, s1, gm.y, bt.y));
                m.z = fmaxf(m.z, in_apply1(v.z, s2, gm.z, bt.z)); m.w = fmaxf(m.w, in_apply1(v.w, s3, gm.w, bt.w));
            }
        }
        *reinterpret_cast<float4*>(out + (((size_t)n * OH + oy) * OW + ox) * C + c4 * 4) = m;
    }
}

// ---------------------------------------------------------------------------------------------------
// K5: pointwise (1x1) convolution as a GEMM:  out[M][N] = act( A[M][K] * W[K][N] + bias (+ residual) )
//   prologue PLAIN : A = in[M][K]
//   prologue GATED : A[m][k] = sum_b gates[crop(m)][b][k] * branch_b[m][k]      for k <  mid
//                            = x[m][k - mid]                                      for k >= mid  (downsample rows)
// CTA: 256 threads, BN output channels (16/32/64), BM = 2048/BN*4 rows; thread = 8 rows x 4 channels;
// K is streamed through shared memory in chunks of 16.
// ---------------------------------------------------------------------------------------------------
struct PwArgs {
    const float* in;          // PLAIN: [M][K];  GATED: x [M][K - mid] (may be null when K == mid)
    const float* branch[4];   // GATED: four [M][mid] tensors
    const float* gates;       // GATED: [crops][4][mid]
    const float* w;           // [K][N]
    const float* bias;        // [N]
    const float* residual;    // [M][N] or null
    float* out;               // [M][N]
    int K, N, mid, HW, relu;
    const float* w_tc;        // canonical hi/lo weight blocks for the tensor-core path (null: CUDA-core kernel)
    int Kpad, Npad;
};

template <int BN, bool GATED>
__global__ void __launch_bounds__(256) k_pointwise(const PwArgs a, const int* __restrict__ d_n, int off, int cap) {
    constexpr int NTN = BN / 4, NTM = 256 / NTN, BM = NTM * 8, BK = 16, LDA = BM + 4;
    const int M = chunk_count(d_n, off, cap) * a.HW;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    if (m0 >= M) return;
    __shared__ __align__(16) float As[BK * LDA];
    __shared__ __align__(16) float Bs[BK * BN];
    const int tn = threadIdx.x % NTN, tm = threadIdx.x / NTN;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const int K = a.K, N = a.N;
    const int KX = GATED ? K - a.mid : 0;
    for (int k0 = 0; k0 < K; k0 += BK) {
        // A chunk: BM rows x 16 k, loaded as float4 along k, stored k-major
        for (int e = threadIdx.x; e < BM * 4; e += 256) {
            const int r = e >> 2, kq = (e & 3) * 4;
            const int m = m0 + r, k = k0 + kq;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < M && k < K) {
                if (!GATED) {
                    v = *reinterpret_cast<const float4*>(a.in + (size_t)m * K + k);
                } else if (k < a.mid) {
                    const float* g = a.gates + (size_t)(m / a.HW) * 4 * a.mid + k;
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        const float4 x = *reinterpret_cast<const float4*>(a.branch[b] + (size_t)m * a.mid + k);
                        const float4 gg = *reinterpret_cast<const float4*>(g + b * a.mid);
                        v.x = fmaf(x.x, gg.x, v.x); v.y = fmaf(x.y, gg.y, v.y);
                        v.z = fmaf(x.z, gg.z, v.z); v.w = fmaf(x.w, gg.w, v.w);
                    }
                } else {
                    v = *reinterpret_cast<const float4*>(a.in + (size_t)m * KX + (k - a.mid));
                }
            }
            As[(kq + 0) * LDA + r] = v.x; As[(kq + 1) * LDA + r] = v.y;
            As[(kq + 2) * LDA + r] = v.z; As[(kq + 3) * LDA + r] = v.w;
        }
        for (int e = threadIdx.x; e < BK * BN / 4; e += 256) {
            const int kk = e / (BN / 4), c = (e % (BN / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k0 + kk < K && n0 + c < N) v = *reinterpret_cast<const float4*>(a.w + (size_t)(k0 + kk) * N + n0 + c);
            *reinterpret_cast<float4*>(Bs + kk * BN + c) = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(As + kk * LDA + tm * 8);
            const float4 a1 = *reinterpret_cast<const float4*>(As + kk * LDA + tm * 8 + 4);
            const float4 b = *reinterpret_cast<const float4*>(Bs + kk * BN + tn * 4);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                acc[i][0] = fmaf(av[i], b.x, acc[i][0]); acc[i][1] = fmaf(av[i], b.y, acc[i][1]);
                acc[i][2] = fmaf(av[i], b.z, acc[i][2]); acc[i][3] = fmaf(av[i], b.w, acc[i][3]);
            }
        }
        __syncthreads();
    }
    const int c = n0 + tn * 4;
    if (c >= N) return;
    const float4 bv = *reinterpret_cast<const float4*>(a.bias + c);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + tm * 8 + i;
        if (m >= M) break;
        float4 v = make_float4(acc[i][0] + bv.x, acc[i][1] + bv.y, acc[i][2] + bv.z, acc[i][3] + bv.w);
        if (a.residual) {
            const float4 r = *reinterpret_cast<const float4*>(a.residual + (size_t)m * N + c);
            v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
        }
        if (a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (a.relu == 2) { v.x = fminf(v.x, 6.f); v.y = fminf(v.y, 6.f); v.z = fminf(v.z, 6.f); v.w = fminf(v.w, 6.f); }  // ReLU6
        *reinterpret_cast<float4*>(a.out + (size_t)m * N + c) = v;
    }
}

// ---------------------------------------------------------------------------------------------------
// K6: LightConv3x3 = 1x1 (linear) -> depthwise 3x3 -> folded BN -> ReLU, fused per spatial tile.
// grid = (row tiles, branches of this level, crops).  Phase A computes T = pw(in) for the tile plus a one-pixel
// halo into shared memory (two pixels x 16 channels per thread per pass, weights broadcast from shared memory);
// phase B applies the depthwise taps from shared memory, writes the activation and, for the last layer of a
// branch, per-tile channel sums for the ChannelGate's global average pool (summed in fixed order later).
// ---------------------------------------------------------------------------------------------------
struct LightArgs {
    const float* in[4];
    float* out[4];
    const float* wpw[4];
    const float* wdw[4];
    const float* bias[4];
    float* sums[4];   // [crops][tiles][C] or null
    int H, W, C, R;   // R = tile rows
    const float* wtc[4];   // 1x1 weights as canonical K-major hi / lo blocks (tc::pack_weights) for the tensor-core stage
};

__global__ void k_lightconv(const LightArgs a, const int* __restrict__ d_n, int off, int cap) {
    const int n = blockIdx.z;
    if (n >= chunk_count(d_n, off, cap)) return;
    const int br = blockIdx.y, tile = blockIdx.x;
    const int H = a.H, W = a.W, C = a.C, R = a.R;
    const int TW = W + 2, TR = R + 2;
    extern __shared__ __align__(16) float smem[];
    float* sT = smem;                       // [TR][TW][C]
    float* sW = sT + (size_t)TR * TW * C;   // [C][C]
    float* sD = sW + (size_t)C * C;         // [9][C]
    float* sP = sD + 9 * C;                 // partial sums [groups][C]
    const int y0 = tile * R;
    const float* in = a.in[br] + (size_t)n * H * W * C;
    for (int e = threadIdx.x; e < C * C; e += blockDim.x) sW[e] = a.wpw[br][e];
    for (int e = threadIdx.x; e < 9 * C; e += blockDim.x) sD[e] = a.wdw[br][e];
    __syncthreads();
    // ---- phase A: T = in * Wpw on the haloed tile ----
    const int n_px = TR * TW;
    const int n_pairs = (n_px + 1) / 2;
    const int n_cchunks = C / 8;  // 8 output channels per pass keeps 16 accumulators for two pixels
    for (int item = threadIdx.x; item < n_pairs * n_cchunks; item += blockDim.x) {
        const int pair = item / n_cchunks, cc = (item - pair * n_cchunks) * 8;
        const int p0 = pair * 2, p1 = p0 + 1;
        const int ty0 = p0 / TW, tx0 = p0 - ty0 * TW;
        const int ty1 = p1 / TW, tx1 = p1 - ty1 * TW;
        const int gy0 = y0 + ty0 - 1, gx0 = tx0 - 1, gy1 = y0 + ty1 - 1, gx1 = tx1 - 1;
        const bool v0 = gy0 >= 0 && gy0 < H && gx0 >= 0 && gx0 < W;
        const bool v1 = p1 < n_px && gy1 >= 0 && gy1 < H && gx1 >= 0 && gx1 < W;
        float acc0[8], acc1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
        if (v0 || v1) {
            const float* q0 = in + ((size_t)gy0 * W + gx0) * C;
            const float* q1 = in + ((size_t)gy1 * W + gx1) * C;
            for (int k = 0; k < C; k += 4) {
                const float4 x0 = v0 ? *reinterpret_cast<const float4*>(q0 + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                const float4 x1 = v1 ? *reinterpret_cast<const float4*>(q1 + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                const float xa[4] = {x0.x, x0.y, x0.z, x0.w};
                const float xb[4] = {x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const float4 w0 = *reinterpret_cast<const float4*>(sW + (size_t)(k + kk) * C + cc);
                    const float4 w1 = *reinterpret_cast<const float4*>(sW + (size_t)(k + kk) * C + cc + 4);
                    acc0[0] = fmaf(xa[kk], w0.x, acc0[0]); acc0[1] = fmaf(xa[kk], w0.y, acc0[1]);
                    acc0[2] = fmaf(xa[kk], w0.z, acc0[2]); acc0[3] = fmaf(xa[kk], w0.w, acc0[3]);
                    acc0[4] = fmaf(xa[kk], w1.x, acc0[4]); acc0[5] = fmaf(xa[kk], w1.y, acc0[5]);
                    acc0[6] = fmaf(xa[kk], w1.z, acc0[6]); acc0[7] = fmaf(xa[kk], w1.w, acc0[7]);
                    acc1[0] = fmaf(xb[kk], w0.x, acc1[0]); acc1[1] = fmaf(xb[kk], w0.y, acc1[1]);
                    acc1[2] = fmaf(xb[kk], w0.z, acc1[2]); acc1[3] = fmaf(xb[kk], w0.w, acc1[3]);
                    acc1[4] = fmaf(xb[kk], w1.x, acc1[4]); acc1[5] = fmaf(xb[kk], w1.y, acc1[5]);
                    acc1[6] = fmaf(xb[kk], w1.z, acc1[6]); acc1[7] = fmaf(xb[kk], w1.w, acc1[7]);
                }
            }
        }
        float4* t0 = reinterpret_cast<float4*>(sT + (size_t)p0 * C + cc);
        t0[0] = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
        t0[1] = make_float4(acc0[4], acc0[5], acc0[6], acc0[7]);
        if (p1 < n_px) {
            float4* t1 = reinterpret_cast<float4*>(sT + (size_t)p1 * C + cc);
            t1[0] = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
            t1[1] = make_float4(acc1[4], acc1[5], acc1[6], acc1[7]);
        }
    }
    __syncthreads();
    // ---- phase B: depthwise 3x3 + bias + ReLU ----
    const int C4 = C / 4;
    const int rows_here = min(R, H - y0);
    const int c4 = threadIdx.x % C4, grp = threadIdx.x / C4, n_grp = blockDim.x / C4;
    float4 wv[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) wv[t] = *reinterpret_cast<const float4*>(sD + t * C + c4 * 4);
    const float4 bv = *reinterpret_cast<const float4*>(a.bias[br] + c4 * 4);
    float4 psum = make_float4(0.f, 0.f, 0.f, 0.f);
    float* outp = a.out[br] + (size_t)n * H * W * C;
    for (int p = grp; p < rows_here * W; p += n_grp) {
        const int y = p / W, x = p - y * W;
        float4 acc = bv;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const float4 t = *reinterpret_cast<const float4*>(sT + ((size_t)(y + ky) * TW + x + kx) * C + c4 * 4);
                const float4 w = wv[ky * 3 + kx];
                acc.x = fmaf(t.x, w.x, acc.x); acc.y = fmaf(t.y, w.y, acc.y);
                acc.z = fmaf(t.z, w.z, acc.z); acc.w = fmaf(t.w, w.w, acc.w);
            }
        acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
        *reinterpret_cast<float4*>(outp + ((size_t)(y0 + y) * W + x) * C + c4 * 4) = acc;
        psum.x += acc.x; psum.y += acc.y; psum.z += acc.z; psum.w += acc.w;
    }
    if (a.sums[br]) {
        *reinterpret_cast<float4*>(sP + (size_t)grp * C + c4 * 4) = psum;
        __syncthreads();
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            float s = 0.f;
            for (int g = 0; g < n_grp; ++g) s += sP[(size_t)g * C + c];
            a.sums[br][((size_t)n * gridDim.x + tile) * C + c] = s;
        }
    }
}

// K6 v2.  Same contract as k_lightconv, restructured around the two limits ncu showed for v1 (L1/TEX 79 %):
//   * phase A read each pixel's K-vector with per-thread float4 loads 64 B apart: every warp request touched 16
//     cache lines.  v2 stages the haloed input tile once with coalesced cp.async into a K-chunk-planar shared
//     layout sX[C/4][pixels] (zero fill outside the image), so phase A reads consecutive float4s (conflict-free),
//     one warp = 64 consecutive pixels x 8 output channels with the 1x1 weights broadcast;
//   * phase B loaded 9 float4 per output from shared memory.  v2 walks columns: a thread owns (x, 4 channels),
//     slides down its rows keeping a 3x3 window in registers and loads 3 float4 per output.
// Shared memory: sX + sT (2 x tile) + weights; pick_tile_rows2 keeps two CTAs per SM for the narrow models.
static inline size_t light2_smem_bytes(int n_px, int C, int threads, int ppl = 4, bool tc_stage = false) {
    const int n_pxp = ((n_px + 32 * ppl - 1) / (32 * ppl)) * (32 * ppl) + 2;
    return sizeof(float) * (2 * (size_t)n_pxp * C + (size_t)C * C * (tc_stage ? 2 : 1) + 9 * C +
                            (size_t)(threads / (C / 4)) * C);
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc));
}

template <int C, int W, int R, int PPL = 4, int MINB = 2, bool TC = false, int NTHREADS = 256>
__global__ void __launch_bounds__(NTHREADS, MINB) k_lightconv2(const LightArgs a, const int* __restrict__ d_n, int off, int cap) {
    const int n = blockIdx.z;
    if (n >= chunk_count(d_n, off, cap)) return;
    const int br = blockIdx.y, tile = blockIdx.x;
    const int H = a.H;
    constexpr int TW = W + 2, TR = R + 2, C4 = C / 4;
    constexpr int n_px = TR * TW;
    constexpr int n_pxp = ((n_px + 32 * PPL - 1) / (32 * PPL)) * (32 * PPL) + 2;   // planes 8 banks apart; whole pixel groups in bounds
    constexpr int NT = NTHREADS;
    extern __shared__ __align__(16) float smem[];
    float4* sX = reinterpret_cast<float4*>(smem);            // [C4][n_pxp]
    float4* sT = sX + (size_t)C4 * n_pxp;                    // [C4][n_pxp]  (planar like sX: conflict-free both ways)
    float* sW = reinterpret_cast<float*>(sT + (size_t)C4 * n_pxp);   // [C][C]
    float* sD = sW + (size_t)C * C;                          // [9][C]
    float* sP = sD + 9 * C;                                  // [NT / C4][C]
    const int y0 = tile * R;
    const float* in = a.in[br] + (size_t)n * H * W * C;
    // ---- stage: weights + haloed input tile (compile-time shapes: the index arithmetic folds to mul/shift) ----
    for (int e = threadIdx.x; e < n_px * C4; e += NT) {
        const int p = e / C4, ch = e - p * C4;
        const int ty = p / TW, tx = p - ty * TW;
        const int gy = y0 + ty - 1, gx = tx - 1;
        float4* dst = sX + ch * n_pxp + p;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) cp_async16(dst, in + ((size_t)gy * W + gx) * C + ch * 4);
        else *dst = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int e = threadIdx.x; e < (n_pxp - n_px) * C4; e += NT) {
        const int q = e / C4, ch = e - q * C4;
        sX[ch * n_pxp + n_px + q] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int e = threadIdx.x; e < C * C / 4; e += NT)
        reinterpret_cast<float4*>(sW)[e] = reinterpret_cast<const float4*>(a.wpw[br])[e];
    for (int e = threadIdx.x; e < 9 * C; e += NT) sD[e] = a.wdw[br][e];
    asm volatile("cp.async.commit_group;");
    asm volatile("cp.async.wait_group 0;");
    if constexpr (TC) {
        // ---- phase A on the tensor cores: T = X * Wpw as wgmma tf32 with the 3-term hi/lo split (float32-class
        // accuracy).  The staged tile IS the canonical no-swizzle K-major operand: a core matrix is 8 consecutive
        // pixels x 16 bytes of one K-chunk plane (contiguous 128 B), the next K chunk is one plane further
        // (LBO = n_pxp * 16 B), the next 8 pixels 128 B further (SBO).  X is split in place (hi) and into the T buffer
        // (lo); each warpgroup takes every other 64-pixel slice and overwrites the lo rows of its slice with T once its
        // own MMAs on them have completed (no other slice reads those rows).
        static_assert(!TC || (C % 16 == 0 && C <= 64), "tensor-core stage: N must be a multiple of 16");
        constexpr int n_ms = (n_px + 63) / 64;
        static_assert(!TC || n_ms * 64 <= n_pxp, "tile rows must stay inside the padded planes");
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        // packed weights (hi block then lo block, canonical [n][k]) over the plain copy in sW: 2 * C * C floats fit
        // because sW + sD + sP follow each other (C*C + 9C + 64C >= 2*C*C for C <= 64)
        __syncthreads();   // cp.async data + the plain sW copy are complete: sW may be overwritten
        float* sWtc = sW;
        for (int e = threadIdx.x; e < 2 * C * C / 4; e += NT)
            reinterpret_cast<float4*>(sWtc)[e] = reinterpret_cast<const float4*>(a.wtc[br])[e];
        // sD was staged before and sits behind sW: re-stage it after the packed weights
        float* sD2 = sWtc + 2 * C * C;
        for (int e = threadIdx.x; e < 9 * C; e += NT) sD2[e] = a.wdw[br][e];
        // split X -> hi (in place) / lo (T buffer), pads included
        for (int e = threadIdx.x; e < C4 * n_pxp; e += NT) {
            const float4 v = sX[e];
            float4 hi, lo;
            hi.x = __uint_as_float(__float_as_uint(v.x) & 0xffffe000u); lo.x = v.x - hi.x;
            hi.y = __uint_as_float(__float_as_uint(v.y) & 0xffffe000u); lo.y = v.y - hi.y;
            hi.z = __uint_as_float(__float_as_uint(v.z) & 0xffffe000u); lo.z = v.z - hi.z;
            hi.w = __uint_as_float(__float_as_uint(v.w) & 0xffffe000u); lo.w = v.w - hi.w;
            sX[e] = hi;
            sT[e] = lo;
        }
        um::fence_async_smem();
        __syncthreads();
        {
            const uint32_t a_hi = um::smem_u32(sX), a_lo = um::smem_u32(sT);
            const uint32_t b_hi = um::smem_u32(sWtc), b_lo = um::smem_u32(sWtc + C * C);
            const uint32_t lbo_a = (uint32_t)n_pxp * 16u, sbo_a = 128u, lbo_b = 128u, sbo_b = (uint32_t)C * 32u;
            const int wg = warp >> 2, row = (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
            float* sTf = reinterpret_cast<float*>(sT);
            for (int u = wg; u < n_ms; u += NT / 128) {
                float acc[TC ? C / 2 : 1];
                um::wg_fence();
#pragma unroll
                for (int ks = 0; ks < C; ks += 8) {
                    const uint32_t ao = (uint32_t)u * 1024u + (uint32_t)(ks >> 2) * lbo_a, bo = (uint32_t)(ks >> 2) * 128u;
                    const uint64_t dah = um::make_desc(a_hi + ao, lbo_a, sbo_a), dal = um::make_desc(a_lo + ao, lbo_a, sbo_a);
                    um::mma<C, true>(acc, dah, b_hi + bo, lbo_b, sbo_b, ks > 0 ? 1u : 0u);
                    um::mma<C, true>(acc, dah, b_lo + bo, lbo_b, sbo_b, 1u);
                    um::mma<C, true>(acc, dal, b_hi + bo, lbo_b, sbo_b, 1u);
                }
                um::wg_commit();
                um::wg_wait_all();
                um::wg_fence_acc<C / 2>(acc);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int p = u * 64 + row + 8 * h;
                    if (p < n_px) {
#pragma unroll
                        for (int i = 0; i < C / 8; ++i) {
                            const int c = 8 * i + cq;
                            *reinterpret_cast<float2*>(sTf + ((size_t)(c >> 2) * n_pxp + p) * 4 + (c & 3)) =
                                make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
                        }
                    }
                }
            }
        }
        __syncthreads();
        sD = sD2;
        sP = sD2 + 9 * C;
    } else {
    __syncthreads();
    // ---- phase A: T = X * Wpw, warp item = (128-pixel group, 8 output channels), 4 pixels per lane ----
    {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        constexpr int G = 32 * PPL;
        constexpr int n_pg = (n_px + G - 1) / G, n_cc = C >> 3;
        for (int item = warp; item < n_pg * n_cc; item += NT / 32) {
            const int pg = item % n_pg, cc = (item / n_pg) * 8;
            const int p0 = pg * G + lane;
            float acc[PPL][8];
#pragma unroll
            for (int q = 0; q < PPL; ++q)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[q][j] = 0.f;
#pragma unroll 2
            for (int kc = 0; kc < C4; ++kc) {
                float xv[PPL][4];
#pragma unroll
                for (int q = 0; q < PPL; ++q) {
                    const float4 x = sX[kc * n_pxp + p0 + 32 * q];
                    xv[q][0] = x.x; xv[q][1] = x.y; xv[q][2] = x.z; xv[q][3] = x.w;
                }
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const float4 w0 = *reinterpret_cast<const float4*>(sW + (kc * 4 + kk) * C + cc);
                    const float4 w1 = *reinterpret_cast<const float4*>(sW + (kc * 4 + kk) * C + cc + 4);
                    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                    for (int q = 0; q < PPL; ++q)
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[q][j] = fmaf(xv[q][kk], wv[j], acc[q][j]);
                }
            }
#pragma unroll
            for (int q = 0; q < PPL; ++q) {
                const int p = p0 + 32 * q;
                if (p < n_px) {
                    sT[(cc / 4) * n_pxp + p] = make_float4(acc[q][0], acc[q][1], acc[q][2], acc[q][3]);
                    sT[(cc / 4 + 1) * n_pxp + p] = make_float4(acc[q][4], acc[q][5], acc[q][6], acc[q][7]);
                }
            }
        }
    }
    __syncthreads();
    }
    // ---- phase B: depthwise 3x3 + bias + ReLU, column walkers with a register window ----
    const int rows_here = min(R, H - y0);
    constexpr int walkers = W * C4;
    constexpr int n_grp = NT / C4;
    constexpr int act = n_grp * C4;    // threads that walk: a multiple of C4 so a thread keeps its channel group
    constexpr int n_split = (act / walkers) < 1 ? 1 : ((act / walkers) > R ? R : (act / walkers));
    constexpr int rows_per = (R + n_split - 1) / n_split;
    float* outp = a.out[br] + (size_t)n * H * W * C;
    float4 psum = make_float4(0.f, 0.f, 0.f, 0.f);
    if (threadIdx.x < act) {
        for (int wk = threadIdx.x; wk < walkers * n_split; wk += act) {
            const int c4 = wk % C4, x = (wk / C4) % W, sp = wk / walkers;
            const int ya = sp * rows_per, yb = min(ya + rows_per, rows_here);
            float4 wv[9];
#pragma unroll
            for (int t = 0; t < 9; ++t) wv[t] = *reinterpret_cast<const float4*>(sD + t * C + c4 * 4);
            const float4 bv = *reinterpret_cast<const float4*>(a.bias[br] + c4 * 4);
            const float4* tbase = sT + c4 * n_pxp + x;
            float4 win[3][3];   // rows (y, y+1, y+2) mod 3 live in fixed registers: the row loop is unrolled by 3
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                win[0][kx] = tbase[ya * TW + kx];
                win[1][kx] = tbase[(ya + 1) * TW + kx];
            }
            float* orow = outp + ((size_t)(y0 + ya) * W + x) * C + c4 * 4;
            for (int y = ya; y < yb; y += 3) {
#pragma unroll
                for (int u = 0; u < 3; ++u) {
                    if (y + u < yb) {
                        const int i0 = u % 3, i1 = (u + 1) % 3, i2 = (u + 2) % 3;
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx)
                            win[i2][kx] = tbase[(y + u + 2) * TW + kx];
                        float4 acc = bv;
#pragma unroll
                        for (int kx = 0; kx < 3; ++kx) {
                            const float4 w0 = wv[kx], w1 = wv[3 + kx], w2 = wv[6 + kx];
                            const float4 t0 = win[i0][kx], t1 = win[i1][kx], t2 = win[i2][kx];
                            acc.x = fmaf(t0.x, w0.x, acc.x); acc.y = fmaf(t0.y, w0.y, acc.y);
                            acc.z = fmaf(t0.z, w0.z, acc.z); acc.w = fmaf(t0.w, w0.w, acc.w);
                            acc.x = fmaf(t1.x, w1.x, acc.x); acc.y = fmaf(t1.y, w1.y, acc.y);
                            acc.z = fmaf(t1.z, w1.z, acc.z); acc.w = fmaf(t1.w, w1.w, acc.w);
                            acc.x = fmaf(t2.x, w2.x, acc.x); acc.y = fmaf(t2.y, w2.y, acc.y);
                            acc.z = fmaf(t2.z, w2.z, acc.z); acc.w = fmaf(t2.w, w2.w, acc.w);
                        }
                        acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f);
                        acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
                        *reinterpret_cast<float4*>(orow + (size_t)u * W * C) = acc;
                        psum.x += acc.x; psum.y += acc.y; psum.z += acc.z; psum.w += acc.w;
                    }
                }
                orow += (size_t)3 * W * C;
            }
        }
    }
    if (a.sums[br]) {
        // every walking thread owns the fixed slot (threadIdx / C4, threadIdx % C4)
        if (threadIdx.x < act)
            *reinterpret_cast<float4*>(sP + (threadIdx.x / C4) * C + (threadIdx.x % C4) * 4) = psum;
        __syncthreads();
        for (int c = threadIdx.x; c < C; c += NT) {
            float s = 0.f;
            for (int g = 0; g < n_grp; ++g) s += sP[g * C + c];
            a.sums[br][((size_t)n * gridDim.x + tile) * C + c] = s;
        }
    }
}

// K6 v3: a whole OSBlock branch (1-4 LightConv3x3 layers) per CTA.  The per-level kernel spends a third of its time
// waiting for its input tile and writes every intermediate level back to HBM; here a CTA stages the conv1 output once
// (tile rows + `depth` halo rows each side), runs  1x1 -> depthwise 3x3 + bias + ReLU  `depth` times between two
// shared-memory buffers (X -> T -> X ...), and only the last level goes to global memory (plus the per-tile channel
// sums for the ChannelGate).  Rows outside the image stay zero in both buffers, which is exactly the zero padding
// every layer of the reference applies; level l only computes the rows level `depth` still needs.
// grid = (row tiles, 4 branches (deepest first), crops); ~12 % redundant halo rows at R = 16, none for full-height tiles.
struct ChainArgs {
    const float* in;        // conv1 output [crops][H][W][C]
    float* out[4];          // final activation of each branch
    const float* wpw[10];   // per LightConv (index = branch*(branch+1)/2 + level-1)
    const float* wdw[10];
    const float* bias[10];
    float* sums[4];         // [crops][tiles][C]
    int H;
};

template <int C, int W, int R, int NT>
__host__ __device__ static constexpr int chain_n_pxp() {
    return (((R + 8) * (W + 2) + 64 + 7) / 8) * 8 + 2;   // room for a trailing 64-pixel group; planes 8 banks apart
}
template <int C, int W, int R, int NT>
static constexpr size_t chain_smem_bytes() {
    return sizeof(float) * ((size_t)2 * chain_n_pxp<C, W, R, NT>() * C + 4 * ((size_t)C * C + 9 * C + C));
}

template <int C, int W, int R, int NT>
__global__ void __launch_bounds__(NT) k_lightchain(const ChainArgs a, const int* __restrict__ d_n, int off, int cap) {
    const int n = blockIdx.z;
    if (n >= chunk_count(d_n, off, cap)) return;
    const int br = 3 - (int)blockIdx.y, depth = br + 1, tile = blockIdx.x;
    const int l0 = br * (br + 1) / 2;
    const int H = a.H;
    constexpr int TW = W + 2, C4 = C / 4, PPL = 2, G = 32 * PPL;   // buffers hold R + 8 padded rows
    constexpr int n_pxp = chain_n_pxp<C, W, R, NT>();
    extern __shared__ __align__(16) float smem[];
    float4* sX = reinterpret_cast<float4*>(smem);     // [C4][n_pxp]  level input (planar: K-chunk major)
    float4* sT = sX + (size_t)C4 * n_pxp;             // [C4][n_pxp]  1x1 result
    float* sW = reinterpret_cast<float*>(sT + (size_t)C4 * n_pxp);   // [4][C][C]
    float* sD = sW + 4 * C * C;                       // [4][9][C]
    float* sB = sD + 4 * 9 * C;                       // [4][C]
    float* sP = reinterpret_cast<float*>(sT);         // [NT / C4][C]  (aliases T: only used after the last level)
    const int y0 = tile * R;
    const int g0 = y0 - 4;                            // global row of local row 0
    const float* in = a.in + (size_t)n * H * W * C;
    // ---- stage: zero both buffers, weights of this branch, the input rows level 1 needs ----
    for (int e = threadIdx.x; e < 2 * C4 * n_pxp; e += NT) sX[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int l = 0; l < depth; ++l) {
        for (int e = threadIdx.x; e < C * C / 4; e += NT)
            reinterpret_cast<float4*>(sW + l * C * C)[e] = reinterpret_cast<const float4*>(a.wpw[l0 + l])[e];
        for (int e = threadIdx.x; e < 9 * C; e += NT) sD[l * 9 * C + e] = a.wdw[l0 + l][e];
        for (int e = threadIdx.x; e < C; e += NT) sB[l * C + e] = a.bias[l0 + l][e];
    }
    __syncthreads();   // the zero fill must land before cp.async writes into the same buffer
    {
        const int ga = max(y0 - depth, 0), gb = min(y0 + R + depth, H);
        const int n_in = (gb - ga) * W * C4;
        for (int e = threadIdx.x; e < n_in; e += NT) {
            const int ch = e % C4, px = e / C4;
            const int gy = ga + px / W, gx = px % W;
            cp_async16(sX + ch * n_pxp + (gy - g0) * TW + gx + 1, in + ((size_t)gy * W + gx) * C + ch * 4);
        }
        asm volatile("cp.async.commit_group;");
        asm volatile("cp.async.wait_group 0;");
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int n_cc = C >> 3;
    constexpr int walkers = W * C4;
    constexpr int n_grp = NT / C4;
    constexpr int act = n_grp * C4;
    constexpr int n_split = (act / walkers) < 1 ? 1 : (act / walkers);
    float4 psum = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int lv = 1; lv <= depth; ++lv) {
        const int ext = depth - lv;                                   // extra rows each side this level still feeds
        const float* w = sW + (lv - 1) * C * C;
        // ---- phase A: T = X * Wpw on image rows [ya-1, yb+1) of this level (whole padded rows) ----
        const int ya = max(y0 - ext, 0), yb = min(y0 + R + ext, H);   // rows phase B produces
        {
            const int ta = max(ya - 1, 0), tb = min(yb + 1, H);
            const int pa = (ta - g0) * TW, pb = (tb - g0) * TW;
            const int n_pg = (pb - pa + G - 1) / G;
            for (int item = warp; item < n_pg * n_cc; item += NT / 32) {
                const int pg = item % n_pg, cc = (item / n_pg) * 8;
                const int p0 = pa + pg * G + lane;
                float acc[PPL][8];
#pragma unroll
                for (int q = 0; q < PPL; ++q)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[q][j] = 0.f;
#pragma unroll 2
                for (int kc = 0; kc < C4; ++kc) {
                    float xv[PPL][4];
#pragma unroll
                    for (int q = 0; q < PPL; ++q) {
                        const float4 x = sX[kc * n_pxp + p0 + 32 * q];
                        xv[q][0] = x.x; xv[q][1] = x.y; xv[q][2] = x.z; xv[q][3] = x.w;
                    }
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const float4 w0 = *reinterpret_cast<const float4*>(w + (kc * 4 + kk) * C + cc);
                        const float4 w1 = *reinterpret_cast<const float4*>(w + (kc * 4 + kk) * C + cc + 4);
                        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                        for (int q = 0; q < PPL; ++q)
#pragma unroll
                            for (int j = 0; j < 8; ++j) acc[q][j] = fmaf(xv[q][kk], wv[j], acc[q][j]);
                    }
                }
#pragma unroll
                for (int q = 0; q < PPL; ++q) {
                    const int p = p0 + 32 * q;
                    if (p < pb) {
                        sT[(cc / 4) * n_pxp + p] = make_float4(acc[q][0], acc[q][1], acc[q][2], acc[q][3]);
                        sT[(cc / 4 + 1) * n_pxp + p] = make_float4(acc[q][4], acc[q][5], acc[q][6], acc[q][7]);
                    }
                }
            }
        }
        __syncthreads();
        // ---- phase B: depthwise 3x3 + bias + ReLU on rows [ya, yb): next level's X, or the branch output ----
        const bool last = lv == depth;
        const int rows_lv = yb - ya;
        const int rows_per = (rows_lv + n_split - 1) / n_split;
        float* outp = a.out[br] + (size_t)n * H * W * C;
        if (threadIdx.x < act) {
            for (int wk = threadIdx.x; wk < walkers * n_split; wk += act) {
                const int c4 = wk % C4, x = (wk / C4) % W, sp = wk / walkers;
                const int ra = ya + sp * rows_per, rb = min(ra + rows_per, yb);
                if (ra >= rb) continue;
                const float* dwp = sD + (lv - 1) * 9 * C + c4 * 4;
                float4 wv[9];
#pragma unroll
                for (int t = 0; t < 9; ++t) wv[t] = *reinterpret_cast<const float4*>(dwp + t * C);
                const float4 bv = *reinterpret_cast<const float4*>(sB + (lv - 1) * C + c4 * 4);
                const float4* tbase = sT + c4 * n_pxp + x;              // column x-1 of the padded row
                float4* xdst = sX + c4 * n_pxp + x + 1;
                float4 win[3][3];
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    win[0][kx] = tbase[(ra - 1 - g0) * TW + kx];
                    win[1][kx] = tbase[(ra - g0) * TW + kx];
                }
                for (int y = ra; y < rb; y += 3) {
#pragma unroll
                    for (int u = 0; u < 3; ++u) {
                        if (y + u < rb) {
                            const int i0 = u % 3, i1 = (u + 1) % 3, i2 = (u + 2) % 3;
#pragma unroll
                            for (int kx = 0; kx < 3; ++kx) win[i2][kx] = tbase[(y + u + 1 - g0) * TW + kx];
                            float4 acc = bv;
#pragma unroll
                            for (int kx = 0; kx < 3; ++kx) {
                                const float4 w0 = wv[kx], w1 = wv[3 + kx], w2 = wv[6 + kx];
                                const float4 t0 = win[i0][kx], t1 = win[i1][kx], t2 = win[i2][kx];
                                acc.x = fmaf(t0.x, w0.x, acc.x); acc.y = fmaf(t0.y, w0.y, acc.y);
                                acc.z = fmaf(t0.z, w0.z, acc.z); acc.w = fmaf(t0.w, w0.w, acc.w);
                                acc.x = fmaf(t1.x, w1.x, acc.x); acc.y = fmaf(t1.y, w1.y, acc.y);
                                acc.z = fmaf(t1.z, w1.z, acc.z); acc.w = fmaf(t1.w, w1.w, acc.w);
                                acc.x = fmaf(t2.x, w2.x, acc.x); acc.y = fmaf(t2.y, w2.y, acc.y);
                                acc.z = fmaf(t2.z, w2.z, acc.z); acc.w = fmaf(t2.w, w2.w, acc.w);
                            }
                            acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f);
                            acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
                            if (last) {
                                *reinterpret_cast<float4*>(outp + ((size_t)(y + u) * W + x) * C + c4 * 4) = acc;
                                psum.x += acc.x; psum.y += acc.y; psum.z += acc.z; psum.w += acc.w;
                            } else {
                                xdst[(y + u - g0) * TW] = acc;
                            }
                        }
                    }
                }
            }
        }
        __syncthreads();
    }
    // per-tile channel sums of the branch output (fixed slot per thread, fixed combination order)
    if (threadIdx.x < act)
        *reinterpret_cast<float4*>(sP + (threadIdx.x / C4) * C + (threadIdx.x % C4) * 4) = psum;
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += NT) {
        float s = 0.f;
        for (int g = 0; g < n_grp; ++g) s += sP[g * C + c];
        a.sums[br][((size_t)n * gridDim.x + tile) * C + c] = s;
    }
}

// K5 v2.  Same contract as k_pointwise.  ncu on v1: long-scoreboard bound (global loads serialised with the math:
// load chunk -> sync -> compute -> sync) and 16 scalar shared stores per thread per chunk for the k-major transpose.
// v2 streams A with cp.async straight into a K-chunk-planar layout As[4][BM] of float4 (rows interleaved over the
// threads so consecutive lanes read consecutive float4: conflict-free, no transpose) and double-buffers the chunks,
// so the copy of chunk c+1 overlaps the FMAs of chunk c.  The GATED prologue (gate-weighted branch sum) still goes
// through registers.
template <int BN, bool GATED, int NT = 256>
__global__ void __launch_bounds__(NT) k_pointwise2(const PwArgs a, const int* __restrict__ d_n, int off, int cap) {
    constexpr int NTN = BN / 4, NTM = NT / NTN, BM = NTM * 8, BK = 16, BMP = BM + 2;
    constexpr int STAGE_F4 = 4 * BMP + BK * BN / 4;   // float4 per stage: A planes + B rows
    const int M = chunk_count(d_n, off, cap) * a.HW;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    if (m0 >= M) return;
    extern __shared__ __align__(16) float4 pw_smem[];
    const int tn = threadIdx.x % NTN, tm = threadIdx.x / NTN;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const int K = a.K, N = a.N;
    const int KX = GATED ? K - a.mid : 0;
    const int n_chunks = (K + BK - 1) / BK;
    auto load_chunk = [&](int c) {
        float4* As = pw_smem + (size_t)(c & 1) * STAGE_F4;
        float4* Bs = As + 4 * BMP;
        const int k0 = c * BK;
        for (int e = threadIdx.x; e < BM * 4; e += NT) {
            const int r = e >> 2, kq = e & 3;
            const int m = m0 + r, k = k0 + kq * 4;
            float4* dst = As + kq * BMP + r;
            if (m < M && k < K) {
                if (!GATED) {
                    cp_async16(dst, a.in + (size_t)m * K + k);
                } else if (k < a.mid) {
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    const float* g = a.gates + (size_t)(m / a.HW) * 4 * a.mid + k;
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        const float4 x = *reinterpret_cast<const float4*>(a.branch[b] + (size_t)m * a.mid + k);
                        const float4 gg = *reinterpret_cast<const float4*>(g + b * a.mid);
                        v.x = fmaf(x.x, gg.x, v.x); v.y = fmaf(x.y, gg.y, v.y);
                        v.z = fmaf(x.z, gg.z, v.z); v.w = fmaf(x.w, gg.w, v.w);
                    }
                    *dst = v;
                } else {
                    cp_async16(dst, a.in + (size_t)m * KX + (k - a.mid));
                }
            } else {
                *dst = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        for (int e = threadIdx.x; e < BK * BN / 4; e += NT) {
            const int kk = e / (BN / 4), c4 = e % (BN / 4);
            if (k0 + kk < K && n0 + c4 * 4 < N) cp_async16(Bs + e, a.w + (size_t)(k0 + kk) * N + n0 + c4 * 4);
            else Bs[e] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        asm volatile("cp.async.commit_group;");
    };
    load_chunk(0);
    for (int c = 0; c < n_chunks; ++c) {
        if (c + 1 < n_chunks) {
            load_chunk(c + 1);
            asm volatile("cp.async.wait_group 1;");
        } else {
            asm volatile("cp.async.wait_group 0;");
        }
        __syncthreads();
        const float4* As = pw_smem + (size_t)(c & 1) * STAGE_F4;
        const float4* Bs = As + 4 * BMP;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
            float xv[8][4];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 x = As[kc * BMP + tm + NTM * i];
                xv[i][0] = x.x; xv[i][1] = x.y; xv[i][2] = x.z; xv[i][3] = x.w;
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float4 b = Bs[(kc * 4 + kk) * (BN / 4) + tn];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    acc[i][0] = fmaf(xv[i][kk], b.x, acc[i][0]); acc[i][1] = fmaf(xv[i][kk], b.y, acc[i][1]);
                    acc[i][2] = fmaf(xv[i][kk], b.z, acc[i][2]); acc[i][3] = fmaf(xv[i][kk], b.w, acc[i][3]);
                }
            }
        }
        __syncthreads();
    }
    const int cn = n0 + tn * 4;
    if (cn >= N) return;
    const float4 bv = *reinterpret_cast<const float4*>(a.bias + cn);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + tm + NTM * i;
        if (m >= M) continue;
        float4 v = make_float4(acc[i][0] + bv.x, acc[i][1] + bv.y, acc[i][2] + bv.z, acc[i][3] + bv.w);
        if (a.residual) {
            const float4 r = *reinterpret_cast<const float4*>(a.residual + (size_t)m * N + cn);
            v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
        }
        if (a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (a.relu == 2) { v.x = fminf(v.x, 6.f); v.y = fminf(v.y, 6.f); v.z = fminf(v.z, 6.f); v.w = fminf(v.w, 6.f); }  // ReLU6
        *reinterpret_cast<float4*>(a.out + (size_t)m * N + cn) = v;
    }
}

// K6b (MobileNetV2): 3x3 stride-2 stem (3 -> C0) + folded BN + ReLU6 : (N,256,128,3) -> (N,128,64,C0)
__global__ void k_stem3(const float* __restrict__ blob, const float* __restrict__ w, const float* __restrict__ bias,
                        int C0, const int* __restrict__ d_n, int off, int cap, float* __restrict__ out) {
    const int n_crops = chunk_count(d_n, off, cap);
    const int C4 = C0 / 4;
    const size_t total = (size_t)n_crops * 128 * 64 * C4;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(e % C4);
        size_t r = e / C4;
        const int ox = (int)(r % 64); r /= 64;
        const int oy = (int)(r % 128);
        const int n = (int)(r / 128);
        float4 acc = *reinterpret_cast<const float4*>(bias + c4 * 4);
        const float* src = blob + (size_t)n * IN_H * IN_W * 3;
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * 2 - 1 + ky;
            if (iy < 0 || iy >= IN_H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * 2 - 1 + kx;
                if (ix < 0 || ix >= IN_W) continue;
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const float a = src[((size_t)iy * IN_W + ix) * 3 + ci];
                    const float4 wv = *reinterpret_cast<const float4*>(w + (size_t)((ky * 3 + kx) * 3 + ci) * C0 + c4 * 4);
                    acc.x = fmaf(a, wv.x, acc.x); acc.y = fmaf(a, wv.y, acc.y);
                    acc.z = fmaf(a, wv.z, acc.z); acc.w = fmaf(a, wv.w, acc.w);
                }
            }
        }
        acc.x = fminf(fmaxf(acc.x, 0.f), 6.f); acc.y = fminf(fmaxf(acc.y, 0.f), 6.f);
        acc.z = fminf(fmaxf(acc.z, 0.f), 6.f); acc.w = fminf(fmaxf(acc.w, 0.f), 6.f);
        *reinterpret_cast<float4*>(out + (((size_t)n * 128 + oy) * 64 + ox) * C0 + c4 * 4) = acc;
    }
}

// K6c (MobileNetV2): depthwise 3x3, stride 1 or 2, pad 1, + folded BN + ReLU6, NHWC float4 channels
__global__ void k_dwconv3(const float* __restrict__ in, int H, int W, int C, int stride, const float* __restrict__ w9c,
                          const float* __restrict__ bias, const int* __restrict__ d_n, int off, int cap,
                          float* __restrict__ out) {
    const int n_crops = chunk_count(d_n, off, cap);
    const int OH = H / stride, OW = W / stride, C4 = C / 4;
    const size_t total = (size_t)n_crops * OH * OW * C4;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(e % C4);
        size_t r = e / C4;
        const int ox = (int)(r % OW); r /= OW;
        const int oy = (int)(r % OH);
        const int n = (int)(r / OH);
        float4 acc = *reinterpret_cast<const float4*>(bias + c4 * 4);
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * stride - 1 + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * stride - 1 + kx;
                if (ix < 0 || ix >= W) continue;
                const float4 v = *reinterpret_cast<const float4*>(in + (((size_t)n * H + iy) * W + ix) * C + c4 * 4);
                const float4 wv = *reinterpret_cast<const float4*>(w9c + (size_t)(ky * 3 + kx) * C + c4 * 4);
                acc.x = fmaf(v.x, wv.x, acc.x); acc.y = fmaf(v.y, wv.y, acc.y);
                acc.z = fmaf(v.z, wv.z, acc.z); acc.w = fmaf(v.w, wv.w, acc.w);
            }
        }
        acc.x = fminf(fmaxf(acc.x, 0.f), 6.f); acc.y = fminf(fmaxf(acc.y, 0.f), 6.f);
        acc.z = fminf(fmaxf(acc.z, 0.f), 6.f); acc.w = fminf(fmaxf(acc.w, 0.f), 6.f);
        *reinterpret_cast<float4*>(out + (((size_t)n * OH + oy) * OW + ox) * C + c4 * 4) = acc;
    }
}

// K7: ChannelGate (osnet.py:161-210): mean -> fc1 -> ReLU -> fc2 -> sigmoid, for the four branches of a block.
struct GateArgs {
    const float* sums[4];  // [crops][tiles][C]
    const float* w1; const float* b1; const float* w2; const float* b2;  // [C][hid], [hid], [hid][C], [C]
    float* gates;          // [crops][4][C]
    int C, hid, tiles, HW;
};
__global__ void k_gates(const GateArgs a, const int* __restrict__ d_n, int off, int cap) {
    const int n = blockIdx.x;
    if (n >= chunk_count(d_n, off, cap)) return;
    extern __shared__ __align__(16) float smem[];
    float* mean = smem;            // [4][C]
    float* hid = smem + 4 * a.C;   // [4][hid]
    const int C = a.C;
    for (int e = threadIdx.x; e < 4 * C; e += blockDim.x) {
        const int b = e / C, c = e - b * C;
        float s = 0.f;
        for (int t = 0; t < a.tiles; ++t) s += a.sums[b][((size_t)n * a.tiles + t) * C + c];
        mean[e] = s / (float)a.HW;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 4 * a.hid; e += blockDim.x) {
        const int b = e / a.hid, h = e - b * a.hid;
        float s = a.b1[h];
        for (int c = 0; c < C; ++c) s = fmaf(mean[b * C + c], a.w1[(size_t)c * a.hid + h], s);
        hid[e] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 4 * C; e += blockDim.x) {
        const int b = e / C, c = e - b * C;
        float s = a.b2[c];
        for (int h = 0; h < a.hid; ++h) s = fmaf(hid[b * a.hid + h], a.w2[(size_t)h * C + c], s);
        a.gates[(size_t)n * 4 * C + e] = 1.0f / (1.0f + expf(-s));
    }
}

// K8: head: global average pool over HW, fc (+ folded BatchNorm1d) + ReLU, row-wise L2 normalisation, scatter
// to the caller's row (base_backend.py:197-207).  One CTA per crop.
__global__ void k_head(const float* __restrict__ x, int HW, int C, const float* __restrict__ wfc,
                       const float* __restrict__ bfc, int FEAT, const CropDesc* __restrict__ crops,
                       const int* __restrict__ d_n, int off, int cap, float* __restrict__ out, int out_ld) {
    const int n = blockIdx.x;
    if (n >= chunk_count(d_n, off, cap)) return;
    extern __shared__ __align__(16) float smem[];
    float* pooled = smem;       // [C]
    float* red = smem + C;      // [32]
    const float* xp = x + (size_t)n * HW * C;
    // global average pool: consecutive threads read consecutive channels of one pixel (coalesced); the pixel
    // stripes of the thread groups are combined in a fixed order so the result is run-to-run deterministic
    float* part = red + 32;  // [groups][C]
    const int groups = blockDim.x / C > 0 ? blockDim.x / C : 1;
    if ((int)threadIdx.x < groups * C) {
        const int c = threadIdx.x % C, g = threadIdx.x / C;
        // four independent partial sums keep several loads in flight (fixed combination order: deterministic)
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        int p = g;
        for (; p + 3 * groups < HW; p += 4 * groups) {
            s0 += xp[(size_t)p * C + c];
            s1 += xp[(size_t)(p + groups) * C + c];
            s2 += xp[(size_t)(p + 2 * groups) * C + c];
            s3 += xp[(size_t)(p + 3 * groups) * C + c];
        }
        for (; p < HW; p += groups) s0 += xp[(size_t)p * C + c];
        part[g * C + c] = (s0 + s1) + (s2 + s3);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        if (blockDim.x >= (unsigned)C) {
            for (int g = 0; g < groups; ++g) s += part[g * C + c];
        } else {
            for (int p = 0; p < HW; ++p) s += xp[(size_t)p * C + c];
        }
        pooled[c] = s / (float)HW;
    }
    __syncthreads();
    float* dst = out + (size_t)crops[off + n].out_row * out_ld;
    float sq = 0.f;
    for (int f = threadIdx.x; f < FEAT; f += blockDim.x) {
        float s;
        if (wfc) {
            // fc + folded BN1d + ReLU; eight independent chains hide the L2 latency of the weight rows
            float t[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            int c = 0;
            for (; c + 8 <= C; c += 8) {
#pragma unroll
                for (int u = 0; u < 8; ++u) t[u] = fmaf(pooled[c + u], wfc[(size_t)(c + u) * FEAT + f], t[u]);
            }
            for (; c < C; ++c) t[0] = fmaf(pooled[c], wfc[(size_t)c * FEAT + f], t[0]);
            s = bfc[f] + (((t[0] + t[1]) + (t[2] + t[3])) + ((t[4] + t[5]) + (t[6] + t[7])));
            s = fmaxf(s, 0.f);
        } else {
            s = pooled[f];  // MobileNetV2: the pooled conv9 map is the embedding (mobilenetv2.py:186-193)
        }
        dst[f] = s;
        sq = fmaf(s, s, sq);
    }
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    const float nrm = sqrtf(tot);
    for (int f = threadIdx.x; f < FEAT; f += blockDim.x) dst[f] = dst[f] / nrm;
}

}  // namespace bmb
#include "lmbn_head.cuh"
#include "vit_small.cuh"   // after every kernel above, whose line numbers (-lineinfo) it leaves unchanged
namespace bmb {

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
enum { CLS_CROP = 0, CLS_STEM, CLS_MAXPOOL, CLS_POINTWISE, CLS_LIGHTCONV, CLS_GATES, CLS_AVGPOOL, CLS_HEAD };
struct LightW { size_t pw, dw, b; };
struct TcW { const float* w = nullptr; int Kpad = 0, Npad = 0; };  // packed weights of one pointwise layer
struct BlockW {
    int cin, cout, mid, hid, has_ds;
    size_t c1w, c1b;
    LightW light[10];
    size_t g1w, g1b, g2w, g2b;
    size_t cw, cb;
    TcW tc_c1, tc_c;
    TcW light_tc[10];   // LightConv 1x1 weights packed for the tensor-core stage (mid % 16 == 0)
    // arch 4: instance norm of the block (IN_NONE / IN_BEFORE_RESIDUAL / IN_AFTER_RESIDUAL), its gamma / beta, and for
    // IN_BEFORE_RESIDUAL with a downsample the downsample's own weights (cw / cb are then conv3 alone)
    int in_mode = 0;
    size_t ing = 0, inb = 0, dsw = 0, dsb = 0;
};
enum { IN_NONE = 0, IN_BEFORE_RESIDUAL = 1, IN_AFTER_RESIDUAL = 2 };

namespace tcx { struct Plan; }

// MobileNetV2 (arch 2): the stem (stem channels, padded to 4), the inverted-residual blocks and conv9
struct MbBlock {
    int cin, cout, t, stride, cinp, midp, coutp;
    size_t we, be, wd, bd, wp, bp;
};
struct MbW {
    int stem = 0, stemp = 0, last = 0;   // last: padded output width of the last block
    size_t stem_w = 0, stem_b = 0, c9w = 0, c9b = 0;
    std::vector<MbBlock> blocks;
};

// LMBN_n (arch 3): OSNet_x1_0 trunk up to conv3[0], three branches (global, partial, channel) of conv3[1:] + conv4 +
// conv5 with their own weights, the bottleneck OSBlock of the global branch, and the neck weights of the head
struct LmbnW {
    BlockW trunk[3];                      // backone.2.0, backone.2.1, backone.3
    size_t trunk_tw = 0, trunk_tb = 0;    // backone.2.2 transition
    BlockW br[3][3];                      // per branch: .0.1, .1.0, .1.1
    size_t br_tw[3] = {0, 0, 0}, br_tb[3] = {0, 0, 0}, br_c5w[3] = {0, 0, 0}, br_c5b[3] = {0, 0, 0};
    BlockW bottleneck;
    size_t neck_w[5] = {0, 0, 0, 0, 0}, neck_b[5] = {0, 0, 0, 0, 0}, sh_w = 0, sh_b = 0, ch_st = 0;
};

// Bottleneck ResNet (arch 5): per convolution the folded bias (offset in d_w) and the tensor-core packing of its weights
struct RnConv { size_t b = 0; const float* w = nullptr; };
struct RnBlock { int cin, width, cout, stride; RnConv c1, c2, c3; };

// MLFN (arch 7): per MLFNBlock the shapes, the tensor-core packings of its dense 1x1 convolutions (FSM layers 1 and 2,
// fm_conv1, fm_conv3, the downsample), and the offsets in d_w of the FSM's last layer and of the grouped 3x3
struct MlfnBlock {
    int cin, cout, mid, gw, f0, f1, stride, ds;
    RnConv fsm1, fsm2, c1, c3, down;
    size_t fsm3w = 0, fsm3b = 0, gcw = 0, gcb = 0;
};
struct MlfnW {
    std::vector<MlfnBlock> blocks;
    RnConv fc_x, fc_s;
};

// HACNN (arch 8): the tensor-core packings of every ConvBlock after the stem (per level the InceptionA's seven, the
// InceptionB's six and the local branch's InceptionB's six, in fold_hacnn's stream order) and of the two heads, and
// the offsets in d_w of each level's attention parameters (sp, w1, b1, w2, b2, wv, bv, wfc, bfc)
struct HacnnW {
    RnConv ia[3][7], ib[3][6], lb[3][6], fcg, fcl;
    size_t att[3][9] = {};
};

// CSPReID-n (arch 10): the tensor-core packings of every ConvBNSiLU after the first stem conv, in fold_cspreid's order
// (stem.1; per stage cv1, each bottleneck's cv1 and cv2, cv2, the stride-2 downsample of stages 1-3; SPPF's cv1 and cv2),
// and the offsets in d_w of the attention's parameters (fc.0, fc.2, depthwise weights, depthwise shift, spatial 1x1) and
// of the three BNNeck3 heads (W, b each)
struct CspW {
    static constexpr int CONVS = 24;
    RnConv conv[CONVS];
    size_t attn[5] = {}, head[6] = {};
};

// CLIP-ReID ViT-B/16 (arch 6): per residual block the offsets in d_w of its LayerNorm parameters and biases, and the
// tensor-core packings of its four linear layers
struct VitLayer {
    size_t ln1g = 0, ln1b = 0, bin = 0, bout = 0, ln2g = 0, ln2b = 0, bfc = 0, bproj = 0;
    const float *win = nullptr, *wout = nullptr, *wfc = nullptr, *wproj = nullptr;
};
struct VitW {
    int tokens = 0, layers = 0;   // 1 + (in_h / 16) (in_w / 16)
    size_t patch_b = 0, pos = 0, lnpre_g = 0, lnpre_b = 0, head_g = 0, head_b = 0, head_w = 0, head_pb = 0;
    const float* patch_w = nullptr;
    std::vector<VitLayer> layer;
};

// ViT-Nano / ViT-Tiny family (arch 9): per block the offsets in d_w of norm1 (LayerNorm gamma, beta; AIN: IN scale,
// LN scale, shift), the biases and norm2, and the tensor-core packings of its four linear layers
struct VitsLayer {
    bool ain = false;
    size_t n1a = 0, n1b = 0, n1c = 0, bqkv = 0, bproj = 0, n2g = 0, n2b = 0, bfc1 = 0, bfc2 = 0;
    const float *wqkv = nullptr, *wproj = nullptr, *wfc1 = nullptr, *wfc2 = nullptr;
};
struct VitsW {
    int tokens = 0, depth = 0, ain = 0, gh = 0, gw = 0, stride = 16, pool = 0, proj = 0;
    size_t patch_b = 0, pos = 0, norm_g = 0, norm_b = 0, head = 0;
    const float* patch_w = nullptr;
    std::vector<VitsLayer> layer;
};

// Backbone of a blob: header word 2, numbered as in weights.py
enum ReidArch {
    ARCH_OSNET = 1,
    ARCH_MOBILENETV2 = 2,
    ARCH_LMBN_N = 3,
    ARCH_OSNET_IN = 4,   // OSNet with instance norms (AIN / IBN)
    ARCH_RESNET = 5,
    ARCH_CLIP = 6,       // CLIP-ReID ViT-B/16
    ARCH_MLFN = 7,
    ARCH_HACNN = 8,
    ARCH_VIT = 9,        // ViT-Nano / ViT-Tiny (vit_nano*, vit_tiny*)
    ARCH_CSPREID = 10,   // CSPReID-n (cspreid_n)
};

struct ReidModel {
    ReidArch arch = ARCH_OSNET;
    int in_h = IN_H;              // crop height
    int in_w = IN_W;              // crop width (256 only for CLIP's vehicle models)
    CropNorm norm = kImageNetNorm;
    VitW vit;
    VitsW vs;
    bool stem_in = false;         // arch 4: conv 7x7 -> IN -> ReLU stem (stem_b is then gamma, stem_beta beta)
    size_t stem_beta = 0;
    float* in_tmp = nullptr;      // arch 4: conv3 output of an IN_BEFORE_RESIDUAL block with a downsample
    LmbnW lm;
    MbW mb;
    std::vector<RnBlock> rn;      // ResNet Bottlenecks, layer1.0 .. layer4.last
    MlfnW ml;
    HacnnW ha;
    CspW cs;
    int* d_n4 = nullptr;          // HACNN: 4 x the crop count, the image count of the [crop][region] local branch
    float* d_wrn = nullptr;       // ResNet / CLIP / MLFN / HACNN / ViT: every GEMM's weights packed by rn::pack_conv_weights
    int c[4] = {0, 0, 0, 0};
    int feat = 0;
    float* d_w = nullptr;
    size_t stem_w = 0, stem_b = 0;
    BlockW blocks[6];
    size_t trans_w[2] = {0, 0}, trans_b[2] = {0, 0};
    size_t c5w = 0, c5b = 0, fcw = 0, fcb = 0;
    TcW tc_trans[2], tc_c5;
    float* d_wtc = nullptr;    // all packed tensor-core weights
    bool use_tc = false;
    int sms = sm_count();   // streaming multiprocessors of the device the model was loaded on (grid sizes)
    bool pw_small = true;   // 128-thread pointwise CTAs; BOXMOT_B200_PW_SMALL=0 for the 256-thread shape
    bool pw_v2 = true;      // BOXMOT_B200_PW_V1=1 selects the first-generation pointwise GEMM (A/B runs)
    bool light_small = false;  // BOXMOT_B200_LIGHT_SMALL=1: stage-2 LightConv as 8-row tiles, 128 threads, 4 CTAs / SM
    bool light_tc = false;     // BOXMOT_B200_LIGHT_TC=1: the stage-2 LightConv 1x1 stage on the tensor cores (tf32 x3)
    bool light_chain = true;   // BOXMOT_B200_LIGHT_CHAIN=0: per-level LightConv launches instead of whole-branch CTAs
    int chain_var = 2;         // BOXMOT_B200_CHAIN_VAR: 2 (default) stage 2 per level + stages 3-4 chained (8-row
                               // stage-2 chain tiles recompute 25 % halo rows); 0 all chained; 1 stage-2 chain
                               // tiles of 16 rows with 512 threads (1 CTA / SM)
    bool light_v2 = true;   // BOXMOT_B200_LIGHT_V1=1 selects the first-generation LightConv kernel (A/B runs)
    // workspace for one chunk of crops
    int chunk = 256;
    float* blob = nullptr;
    float* bufA = nullptr;
    float* bufB = nullptr;
    float* x1 = nullptr;
    float* Y[4][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};
    float* sums[4] = {nullptr, nullptr, nullptr, nullptr};
    float* gates = nullptr;
    float* trunk = nullptr;    // LMBN_n: trunk output, read by all three branches
    float* pooled = nullptr;   // LMBN_n: [crops][6][512] head poolings
    // per-kernel-class device timing (bench / profiles): events around every launch when enabled
    bool profile = false;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int> prof_cls;
    double prof_ms[REID_N_CLASSES] = {0};
    int prof_launches[REID_N_CLASSES] = {0};
    int preprocess = 0;        // 0 resize, 1 resize_pad
    tcx::Plan* tc = nullptr;   // tensor-core path (wgmma + TMA, reid_tc.cuh): the default for the widths it covers
    int debug_stop = -1;       // stop after this stage index and leave the tensor in debug_ptr
    const float* debug_ptr = nullptr;
    size_t debug_floats_per_crop = 0;
};

static const int kBranchOfLight[10] = {0, 1, 1, 2, 2, 2, 3, 3, 3, 3};
static const int kLevelOfLight[10] = {1, 1, 2, 1, 2, 3, 1, 2, 3, 4};
static const int kDepth[4] = {1, 2, 3, 4};

}  // namespace bmb
#include "reid_tc_host.cuh"
namespace bmb {
namespace tcx {
Plan* plan_build(ReidModel* m, const float* host_w);
bool plan_supported(const ReidModel* m);
}

namespace {
// Offsets of the tensors in the blob payload, in walk order; every tensor starts 16-byte aligned
struct BlobCursor {
    size_t o = 0;
    size_t operator()(size_t n) { const size_t r = o; o += (n + 3) / 4 * 4; return r; }
};

// Layers whose K-major [K][N] weights rn::k_conv_tc reads pre-split (rn::pack_conv_weights): ResNet's convolutions and
// CLIP's linear layers.  The layout queues them; after the upload each `dst` points at its packing in m->d_wrn.
struct WgmmaPack {
    struct Todo { const float** dst; size_t w; int K, N; size_t at; };
    std::vector<Todo> todo;
    size_t n = 0;
    void add(const float*& dst, size_t w, int K, int N) {
        todo.push_back({&dst, w, K, N, n});
        n += 2 * (size_t)K * N;
    }
};

// Per-crop float counts of the workspace buffers a chunk runner uses (0: not allocated)
struct Workspace {
    size_t blob = 0, bufA = 0, bufB = 0, x1 = 0, Y[4][2] = {}, sums[4] = {}, gates = 0, trunk = 0, pooled = 0, in_tmp = 0;
    size_t total() const {
        size_t t = blob + bufA + bufB + x1 + gates + trunk + pooled + in_tmp;
        for (int b = 0; b < 4; ++b) t += Y[b][0] + Y[b][1] + sums[b];
        return t;
    }
};

// The arch-specific header words: the model's geometry, checked before the payload is read
void read_header(ReidModel* m, const int32_t* hdr) {
    m->arch = (ReidArch)hdr[2];
    m->feat = hdr[7];
    switch (m->arch) {
        case ARCH_CLIP:
            if (hdr[3] != vit::D || hdr[4] < 1 || hdr[4] > 64 || hdr[5] != vit::HEADS || hdr[6] != vit::PROJ ||
                hdr[7] != vit::FEAT)
                throw std::runtime_error("bad CLIP blob header (only ViT-B/16: width 768, 12 heads, 512-d projection)");
            m->in_h = hdr[9];
            m->in_w = hdr[10];
            if (m->in_h != 256 || (m->in_w != 128 && m->in_w != 256) || hdr[11] != m->in_h / vit::PATCH ||
                hdr[12] != m->in_w / vit::PATCH)
                throw std::runtime_error("bad CLIP blob header (input 256x128 or 256x256, 16x16 patches)");
            m->norm = CropNorm{{0.5f, 0.5f, 0.5f}, {0.5f, 0.5f, 0.5f}};
            m->vit.layers = hdr[4];
            m->vit.tokens = 1 + hdr[11] * hdr[12];
            return;
        case ARCH_VIT: {
            // words 3-7: width, depth, heads, AIN blocks, row width; 9-15: crop h, w, grid h, w, patch stride,
            // pooling (0 class token, 1 omni-scale, P >= 2 class token + P strips), projection width (0 or 512)
            VitsW& v = m->vs;
            v.depth = hdr[4]; v.ain = hdr[6];
            m->in_h = hdr[9]; m->in_w = hdr[10];
            v.gh = hdr[11]; v.gw = hdr[12]; v.stride = hdr[13]; v.pool = hdr[14]; v.proj = hdr[15];
            v.tokens = 1 + v.gh * v.gw;
            const bool geom = m->in_h >= 16 && m->in_h <= IN_H_MAX && m->in_w == IN_W && (v.stride == 16 || v.stride == 12) &&
                              v.gh == (m->in_h - vit::PATCH) / v.stride + 1 && v.gw == (m->in_w - vit::PATCH) / v.stride + 1 &&
                              v.tokens <= vits::MAX_T;
            const bool head = (v.proj == 0 || v.proj == vits::PROJ) && v.pool >= 0 && v.pool <= vits::MAX_PARTS &&
                              (v.pool != 1 || (v.proj == 0 && v.gh % 8 == 0)) && (v.pool < 2 || (v.proj && v.pool <= v.gh)) &&
                              m->feat == vits::head_feat(v.pool, v.proj);
            if (hdr[3] != vits::D || hdr[5] != vits::HEADS || v.depth < 1 || v.depth > 64 || v.ain < 0 ||
                v.ain > v.depth || !geom || !head || (v.ain && vits::ain_smem_bytes(v.tokens) > 200 * 1024))
                throw std::runtime_error("bad ViT blob header (width 192, 3 heads, 16x16 patches at stride 16 or 12, "
                                         "at most 320 tokens, a known pooling head)");
            return;
        }
        case ARCH_MLFN:
            if (hdr[3] != 64 || hdr[4] != 2048 || hdr[5] != mlfn::GROUPS || hdr[6] != mlfn::BLOCKS || m->feat != mlfn::FEAT)
                throw std::runtime_error("bad MLFN blob header (only groups 32, channels 64-2048, 16 blocks, 1024-d)");
            m->c[0] = 64;
            return;
        case ARCH_CSPREID:
            // words 3-7: stage widths 128, 256, 384, 512 and the 1536-d row; 9-10: crop h, w (256x128 or 256x256)
            if (hdr[3] != 128 || hdr[4] != 256 || hdr[5] != 384 || hdr[6] != csp::C || m->feat != csp::FEAT ||
                hdr[9] != 256 || (hdr[10] != 128 && hdr[10] != 256))
                throw std::runtime_error("bad CSPReID-n blob header (only widths 128/256/384/512, 1536-d, 256x128 or "
                                         "256x256 input)");
            m->in_h = hdr[9];
            m->in_w = hdr[10];
            return;
        case ARCH_HACNN:
            if (hdr[3] != hacnn::STEM_C || hdr[4] != 128 || hdr[5] != 256 || hdr[6] != hacnn::C3 ||
                m->feat != hacnn::FEAT || hdr[9] != hacnn::IN_H || hdr[10] != hacnn::IN_W)
                throw std::runtime_error("bad HACNN blob header (only nchannels 128/256/384, 1024-d, 160x64 input)");
            m->in_h = hacnn::IN_H;
            m->in_w = hacnn::IN_W;
            return;
        case ARCH_RESNET:
            m->c[0] = 64;
            for (int l = 0; l < 4; ++l)
                if (hdr[3 + l] < 1 || hdr[3 + l] > 64) throw std::runtime_error("bad ResNet blob header (block counts)");
            if (m->feat != 2048) throw std::runtime_error("bad ResNet blob header (feature dim)");
            return;
        case ARCH_MOBILENETV2:   // hdr[4] blocks: it sizes the block table that follows the header
            m->mb.stem = hdr[3];
            m->mb.stemp = (hdr[3] + 3) / 4 * 4;
            if (hdr[4] < 1 || hdr[4] > 64 || m->feat < 1) throw std::runtime_error("bad MobileNetV2 blob header");
            return;
        case ARCH_OSNET:
        case ARCH_LMBN_N:
        case ARCH_OSNET_IN:
            for (int i = 0; i < 4; ++i) m->c[i] = hdr[3 + i];
            if (m->c[0] % 16 != 0 || m->feat < 1) throw std::runtime_error("unsupported OSNet width (stem channels)");
            if (m->arch == ARCH_LMBN_N) {
                if (hdr[9] != 384 || m->c[0] != 64 || m->c[1] != 256 || m->c[2] != 384 || m->c[3] != LMBN_C ||
                    m->feat != LMBN_VECS * LMBN_C)
                    throw std::runtime_error("unsupported LMBN_n blob header (expected 384x128 input, widths 64/256/384/512, 3584-d)");
                m->in_h = hdr[9];
            }
            if (m->arch == ARCH_OSNET_IN) {   // header word 9: stem IN flag; words 10-15: per-block IN placement
                m->stem_in = hdr[9] != 0;
                for (int i = 0; i < 6; ++i)
                    if (hdr[10 + i] < IN_NONE || hdr[10 + i] > IN_AFTER_RESIDUAL)
                        throw std::runtime_error("bad instance-norm placement in an arch-4 ReID blob header");
            }
            return;
    }
}

// OSNet-family workspace per crop at crop height in_h: the crop, two block maps as large as the stem output
// (in_h/2 x 64 x c0) or the stage-2 maps (in_h/4 x 32 x c1), whichever is larger, the conv1 output and the eight
// LightConv maps of a stage-2 block, the branch sums and gates, and for LMBN_n the trunk output and the head poolings
Workspace osnet_workspace(const ReidModel* m, int in_h, bool lmbn) {
    Workspace ws;
    const size_t big = std::max((size_t)(in_h / 2) * 64 * m->c[0], (size_t)(in_h / 4) * 32 * m->c[1]);
    const size_t mid = (size_t)(in_h / 4) * 32 * (m->c[1] / 4);
    ws.blob = (size_t)in_h * IN_W * 3;
    ws.bufA = ws.bufB = big;
    ws.x1 = mid;
    for (int b = 0; b < 4; ++b) {
        ws.Y[b][0] = ws.Y[b][1] = mid;
        ws.sums[b] = 64 * (size_t)(m->c[3] / 4);
    }
    ws.gates = 4 * (size_t)(m->c[3] / 4);
    if (lmbn) {
        ws.trunk = (size_t)(in_h / 8) * 16 * m->c[2];
        ws.pooled = (size_t)LMBN_POOLS * LMBN_C;
    }
    return ws;
}

// ---- OSNet, LMBN_n and OSNet-AIN / IBN (arch 1, 3, 4): stem, OSBlocks, transitions, conv5 and fc (or LMBN_n's
// branches and neck) ----
Workspace layout_osnet(ReidModel* m, const int32_t* hdr, BlobCursor& take) {
    auto take_block = [&](BlockW& b, int cin, int cout, int in_mode = IN_NONE) {
        b.in_mode = in_mode;
        b.cin = cin;
        b.cout = cout;
        b.mid = b.cout / 4;
        b.hid = b.mid / 16;
        b.has_ds = b.cin != b.cout;
        if (b.mid % 8 != 0 || b.hid < 1) throw std::runtime_error("unsupported OSNet width (mid channels)");
        b.c1w = take((size_t)b.cin * b.mid);
        b.c1b = take(b.mid);
        for (int l = 0; l < 10; ++l) {
            b.light[l].pw = take((size_t)b.mid * b.mid);
            b.light[l].dw = take((size_t)9 * b.mid);
            b.light[l].b = take(b.mid);
        }
        b.g1w = take((size_t)b.mid * b.hid);
        b.g1b = take(b.hid);
        b.g2w = take((size_t)b.hid * b.mid);
        b.g2b = take(b.mid);
        if (in_mode == IN_BEFORE_RESIDUAL) {   // conv3 alone (zero bias), then the downsample on its own
            b.cw = take((size_t)b.mid * b.cout);
            b.cb = take(b.cout);
            if (b.has_ds) {
                b.dsw = take((size_t)b.cin * b.cout);
                b.dsb = take(b.cout);
            }
        } else {
            b.cw = take((size_t)(b.mid + (b.has_ds ? b.cin : 0)) * b.cout);
            b.cb = take(b.cout);
        }
        if (in_mode != IN_NONE) {
            if (b.cout % 4) throw std::runtime_error("unsupported OSNet width (instance-norm channels)");
            b.ing = take(b.cout);
            b.inb = take(b.cout);
        }
    };
    m->stem_w = take((size_t)147 * m->c[0]);
    m->stem_b = take(m->c[0]);
    if (m->stem_in) m->stem_beta = take(m->c[0]);
    if (m->arch == ARCH_LMBN_N) {   // weights.fold_lmbn_n walk order
        LmbnW& lm = m->lm;
        take_block(lm.trunk[0], 64, 256);
        take_block(lm.trunk[1], 256, 256);
        lm.trunk_tw = take((size_t)256 * 256);
        lm.trunk_tb = take(256);
        take_block(lm.trunk[2], 256, 384);
        for (int br = 0; br < 3; ++br) {
            take_block(lm.br[br][0], 384, 384);
            lm.br_tw[br] = take((size_t)384 * 384);
            lm.br_tb[br] = take(384);
            take_block(lm.br[br][1], 384, 512);
            take_block(lm.br[br][2], 512, 512);
            lm.br_c5w[br] = take((size_t)512 * 512);
            lm.br_c5b[br] = take(512);
        }
        take_block(lm.bottleneck, 512, 512);
        for (int k = 0; k < 5; ++k) {
            lm.neck_w[k] = take((size_t)LMBN_C * LMBN_C);
            lm.neck_b[k] = take(LMBN_C);
        }
        lm.sh_w = take((size_t)(LMBN_C / 2) * LMBN_C);
        lm.sh_b = take(LMBN_C);
        lm.ch_st = take((size_t)4 * LMBN_C);
        return osnet_workspace(m, m->in_h, true);
    }
    for (int s = 0; s < 3; ++s) {
        for (int j = 0; j < 2; ++j)
            take_block(m->blocks[s * 2 + j], j == 0 ? m->c[s] : m->c[s + 1], m->c[s + 1],
                       m->arch == ARCH_OSNET_IN ? hdr[10 + s * 2 + j] : IN_NONE);
        if (s < 2) {
            m->trans_w[s] = take((size_t)m->c[s + 1] * m->c[s + 1]);
            m->trans_b[s] = take(m->c[s + 1]);
        }
    }
    m->c5w = take((size_t)m->c[3] * m->c[3]);
    m->c5b = take(m->c[3]);
    m->fcw = take((size_t)m->c[3] * m->feat);
    m->fcb = take(m->feat);
    Workspace ws = osnet_workspace(m, m->in_h, false);
    // arch 4: the instance-norm statistics ({mean, rstd} per crop and channel, 4 floats) live in sums[0], which
    // holds 16 * c3 >= 4 * C floats per crop and is free whenever they are needed (the stem runs before any block;
    // a block's norm follows its gates kernel, the last reader of the branch sums).  The one extra buffer is the
    // conv3 output of an IN_BEFORE_RESIDUAL block whose downsample GEMM writes the block output.
    for (const BlockW& b : m->blocks)
        if (b.in_mode == IN_BEFORE_RESIDUAL && b.has_ds) ws.in_tmp = ws.bufA;
    return ws;
}

// ---- MobileNetV2 (reid/backbones/mobilenetv2.py): stem, 17 inverted-residual blocks, conv9, GAP ----
// table: cin, cout, expansion, stride of every block
Workspace layout_mobilenetv2(ReidModel* m, const std::vector<int32_t>& table, BlobCursor& take) {
    MbW& mb = m->mb;
    auto p4 = [](int n) { return (n + 3) / 4 * 4; };
    mb.stem_w = take((size_t)27 * mb.stemp);
    mb.stem_b = take(mb.stemp);
    int H = 128, Wd = 64;
    size_t max_x = (size_t)H * Wd * mb.stemp, max_e = 0, max_d = 0;
    for (size_t i = 0; i < table.size(); i += 4) {
        MbBlock b{};
        b.cin = table[i]; b.cout = table[i + 1]; b.t = table[i + 2]; b.stride = table[i + 3];
        if (b.stride != 1 && b.stride != 2) throw std::runtime_error("bad MobileNetV2 stride");
        b.cinp = p4(b.cin); b.midp = p4(b.cin * b.t); b.coutp = p4(b.cout);
        b.we = take((size_t)b.cinp * b.midp); b.be = take(b.midp);
        b.wd = take((size_t)9 * b.midp); b.bd = take(b.midp);
        b.wp = take((size_t)b.midp * b.coutp); b.bp = take(b.coutp);
        max_e = std::max(max_e, (size_t)H * Wd * b.midp);
        H /= b.stride; Wd /= b.stride;
        max_d = std::max(max_d, (size_t)H * Wd * b.midp);
        max_x = std::max(max_x, (size_t)H * Wd * b.coutp);
        mb.blocks.push_back(b);
    }
    mb.last = mb.blocks.back().coutp;
    const int featp = p4(m->feat);
    mb.c9w = take((size_t)mb.last * featp);
    mb.c9b = take(featp);
    if (featp != m->feat) throw std::runtime_error("ReID blob size does not match its header");
    // per crop: the crop, two block maps, the expansion output and the depthwise output, each at its largest
    Workspace ws;
    ws.blob = (size_t)m->in_h * m->in_w * 3;
    ws.bufA = ws.bufB = std::max(max_x, (size_t)H * Wd * featp);
    ws.x1 = max_e;
    ws.Y[0][0] = max_d;
    return ws;
}

// ---- Bottleneck ResNet (reid/backbones/resnet.py resnet50 / resnet101): stem, layer1..4, GAP ----
Workspace layout_resnet(ReidModel* m, const int32_t* hdr, BlobCursor& take, WgmmaPack& pack) {
    m->stem_w = take((size_t)147 * 64);
    m->stem_b = take(64);
    auto conv = [&](RnConv& c, int K, int N) {
        const size_t w = take((size_t)K * N);
        c.b = take(N);
        pack.add(c.w, w, K, N);
    };
    int cin = 64;
    m->rn.reserve((size_t)hdr[3] + hdr[4] + hdr[5] + hdr[6]);   // `pack` keeps pointers into the blocks
    for (int l = 0; l < 4; ++l)
        for (int j = 0; j < hdr[3 + l]; ++j) {
            RnBlock b{};
            b.cin = cin; b.width = 64 << l; b.cout = 4 * b.width; b.stride = (j == 0 && l > 0) ? 2 : 1;
            m->rn.push_back(b);
            RnBlock& r = m->rn.back();
            conv(r.c1, r.cin, r.width);
            conv(r.c2, 9 * r.width, r.width);
            conv(r.c3, r.width + (j == 0 ? r.cin : 0), r.cout);
            cin = r.cout;
        }
    if (cin != m->feat) throw std::runtime_error("ReID blob size does not match its header");
    // per crop: the staged crop, two block maps as large as the stem output / layer1's 64x32x256, layer2.0's
    // conv1 output (64x32x128) and layer1's conv2 output (64x32x64): 1.54 M floats, below the 2.36 M an
    // OSNet_x1_0 chunk takes per crop, so the chunk keeps its size
    Workspace ws;
    ws.blob = (size_t)m->in_h * m->in_w * 3;
    ws.bufA = ws.bufB = (size_t)128 * 64 * 64;
    ws.x1 = (size_t)64 * 32 * 128;
    ws.Y[0][0] = (size_t)64 * 32 * 64;
    return ws;
}

// ---- MLFN (reid/backbones/mlfn.py): stem, 16 MLFNBlocks, fc_x / fc_s head ----
Workspace layout_mlfn(ReidModel* m, BlobCursor& take, WgmmaPack& pack) {
    static const int kStages[4][4] = {{3, 256, 128, 64}, {4, 512, 256, 128}, {6, 1024, 512, 128}, {3, 2048, 512, 128}};
    m->stem_w = take((size_t)147 * 64);
    m->stem_b = take(64);
    auto conv = [&](RnConv& c, int K, int N) {
        const size_t w = take((size_t)K * N);
        c.b = take(N);
        pack.add(c.w, w, K, N);
    };
    MlfnW& ml = m->ml;
    ml.blocks.reserve(mlfn::BLOCKS);   // `pack` keeps pointers into the blocks
    int cin = 64;
    for (int s = 0; s < 4; ++s)
        for (int j = 0; j < kStages[s][0]; ++j) {
            MlfnBlock b{};
            b.cin = cin; b.cout = kStages[s][1]; b.mid = b.cout / 2; b.gw = b.mid / mlfn::GROUPS;
            b.f0 = kStages[s][2]; b.f1 = kStages[s][3];
            b.stride = (j == 0 && s > 0) ? 2 : 1;
            b.ds = b.cin != b.cout || b.stride > 1;
            ml.blocks.push_back(b);
            MlfnBlock& r = ml.blocks.back();
            conv(r.fsm1, r.cin, r.f0);
            conv(r.fsm2, r.f0, r.f1);
            r.fsm3w = take((size_t)r.f1 * mlfn::GROUPS);
            r.fsm3b = take(mlfn::GROUPS);
            conv(r.c1, r.cin, r.mid);
            r.gcw = take((size_t)9 * r.gw * r.mid);
            r.gcb = take(r.mid);
            conv(r.c3, r.mid, r.cout);
            if (r.ds) conv(r.down, r.cin, r.cout);
            cin = r.cout;
        }
    conv(ml.fc_x, 2048, mlfn::FEAT);
    conv(ml.fc_s, mlfn::SHAT, mlfn::FEAT);
    // per crop: the staged crop, two block maps as large as the stem output / stage 1's 64x32x256, fm_conv1's output
    // (at most 64x32x256, the first block of stage 2), fm_conv2's (at most 64x32x128), and rows for the pooled map
    // (2048), s_hat (512), the FSM hidden layers (512, 128), fc_x and x + s (1024 each): 1.94 M floats, below the
    // 2.36 M an OSNet_x1_0 chunk takes per crop, so the chunk keeps its size.  The downsample writes the block output
    // buffer, which fm_conv3 then reads as its residual and overwrites in place.
    Workspace ws;
    ws.blob = (size_t)m->in_h * m->in_w * 3;
    ws.bufA = ws.bufB = (size_t)128 * 64 * 64;
    ws.x1 = (size_t)64 * 32 * 256;
    ws.Y[0][0] = (size_t)64 * 32 * 128;
    ws.pooled = 2048;
    ws.gates = mlfn::SHAT;
    ws.sums[0] = 512;
    ws.sums[1] = 128;
    ws.sums[2] = ws.sums[3] = mlfn::FEAT;
    return ws;
}

// ---- HACNN (reid/backbones/hacnn.py): stem, three Inception + HarmAttn levels, the local branch, two heads ----
Workspace layout_hacnn(ReidModel* m, BlobCursor& take, WgmmaPack& pack) {
    static const int kC[4] = {hacnn::STEM_C, 128, 256, hacnn::C3};
    m->stem_w = take((size_t)27 * hacnn::STEM_C);
    m->stem_b = take(hacnn::STEM_C);
    auto conv = [&](RnConv& c, int K, int N) {
        const size_t w = take((size_t)K * N);
        c.b = take(N);
        pack.add(c.w, w, K, N);
    };
    auto inception_b = [&](RnConv* cv, int cin, int cout) {
        const int mid = cout / 4;
        conv(cv[0], cin, mid);
        conv(cv[1], 9 * mid, mid);
        conv(cv[2], cin, mid);
        conv(cv[3], 9 * mid, mid);
        conv(cv[4], 9 * mid, mid);
        conv(cv[5], cin, 2 * mid);
    };
    HacnnW& h = m->ha;
    for (int i = 0; i < 3; ++i) {
        const int cin = kC[i], c = kC[i + 1], mid = c / 4, r = c / 16;
        for (int s = 0; s < 3; ++s) {
            conv(h.ia[i][2 * s], cin, mid);
            conv(h.ia[i][2 * s + 1], 9 * mid, mid);
        }
        conv(h.ia[i][6], cin, mid);
        inception_b(h.ib[i], c, c);
        const size_t sizes[9] = {12, (size_t)c * r, (size_t)r, (size_t)r * c, (size_t)c, (size_t)c * c, (size_t)c,
                                 (size_t)c * 8, 8};
        for (int k = 0; k < 9; ++k) h.att[i][k] = take(sizes[k]);
    }
    for (int i = 0; i < 3; ++i) inception_b(h.lb[i], kC[i], kC[i + 1]);
    conv(h.fcg, hacnn::C3, hacnn::HALF);
    conv(h.fcl, 4 * hacnn::C3, hacnn::HALF);
    // per crop: the crop; two maps as large as the stem output (80x32x32, also x1_out 40x16x128) for the previous and
    // the current level; InceptionA's output (at most 80x32x128); three stream scratch maps and the local branch's
    // STN map and local map (each at most 4 x 24x28x32); the attention's s (40x16) and v (384), theta (24), the two
    // heads' pools (384 + 1536) and the head row (1024): 0.96 M floats, below OSNet_x1_0's 2.36 M, so the chunk keeps
    // its size.
    constexpr size_t kLocal = (size_t)4 * 24 * 28 * 32;
    Workspace ws;
    ws.blob = (size_t)hacnn::IN_H * hacnn::IN_W * 3;
    ws.bufA = ws.bufB = (size_t)80 * 32 * 32;
    ws.x1 = (size_t)80 * 32 * 128;
    ws.Y[0][0] = ws.Y[0][1] = ws.Y[1][0] = ws.Y[1][1] = ws.Y[2][0] = kLocal;
    ws.sums[0] = hacnn::MAX_HW;
    ws.sums[1] = hacnn::MAX_C;
    ws.sums[2] = hacnn::FEAT;
    ws.gates = hacnn::THETA;
    ws.pooled = 5 * hacnn::C3;
    return ws;
}

// ---- CLIP-ReID ViT-B/16 (reid/backbones/clip): patch embedding, ln_pre, 12 residual attention blocks, head ----
Workspace layout_clip(ReidModel* m, BlobCursor& take, WgmmaPack& pack) {
    constexpr int D = vit::D;
    VitW& v = m->vit;
    auto linear = [&](const float*& dst, int K, int N) { pack.add(dst, take((size_t)K * N), K, N); };
    linear(v.patch_w, 3 * vit::PATCH * vit::PATCH, D);
    v.patch_b = take(D);
    v.pos = take((size_t)v.tokens * D);
    v.lnpre_g = take(D); v.lnpre_b = take(D);
    v.layer.resize(v.layers);   // `pack` keeps pointers into the layers
    for (VitLayer& l : v.layer) {
        l.ln1g = take(D); l.ln1b = take(D);
        linear(l.win, D, 3 * D); l.bin = take(3 * D);
        linear(l.wout, D, D); l.bout = take(D);
        l.ln2g = take(D); l.ln2b = take(D);
        linear(l.wfc, D, 4 * D); l.bfc = take(4 * D);
        linear(l.wproj, 4 * D, D); l.bproj = take(D);
    }
    v.head_g = take(D); v.head_b = take(D);
    v.head_w = take((size_t)D * vit::PROJ); v.head_pb = take(vit::PROJ);
    // per crop: the staged crop, the residual stream, the LayerNorm output and the attention output
    // ([T][768] each), q | k | v ([T][2304]) and the MLP hidden layer ([T][3072], which also holds the patch
    // rows): 1.09 M floats at 129 tokens, 2.17 M at 257, both below the 2.36 M an OSNet_x1_0 chunk takes per
    // crop, so the chunk keeps its size
    const size_t T = v.tokens;
    Workspace ws;
    ws.blob = (size_t)m->in_h * m->in_w * 3;
    ws.bufA = ws.bufB = ws.Y[0][0] = T * D;
    ws.x1 = T * 3 * D;
    ws.Y[0][1] = T * 4 * D;
    return ws;
}

// ---- ViT-Nano / ViT-Tiny (reid/backbones/vit_nano.py, vit_tiny.py): patch embedding, tokens, blocks, norm, head ----
Workspace layout_vits(ReidModel* m, BlobCursor& take, WgmmaPack& pack) {
    constexpr int D = vits::D;
    VitsW& v = m->vs;
    auto linear = [&](const float*& dst, int K, int N) { pack.add(dst, take((size_t)K * N), K, N); };
    linear(v.patch_w, 3 * vit::PATCH * vit::PATCH, D);
    v.patch_b = take(D);
    v.pos = take((size_t)v.tokens * D);
    v.layer.resize(v.depth);   // `pack` keeps pointers into the layers
    for (int i = 0; i < v.depth; ++i) {
        VitsLayer& l = v.layer[i];
        l.ain = i < v.ain;
        l.n1a = take(D); l.n1b = take(D);
        if (l.ain) l.n1c = take(D);
        linear(l.wqkv, D, 3 * D); l.bqkv = take(3 * D);
        linear(l.wproj, D, D); l.bproj = take(D);
        l.n2g = take(D); l.n2b = take(D);
        linear(l.wfc1, D, vits::MLP); l.bfc1 = take(vits::MLP);
        linear(l.wfc2, vits::MLP, D); l.bfc2 = take(D);
    }
    v.norm_g = take(D); v.norm_b = take(D);
    v.head = take(vits::head_floats(v.pool, v.proj));
    // per crop: the staged crop, the residual stream, the norm output and the attention output ([T][192] each),
    // q | k | v ([T][576], also the head tap) and the MLP hidden layer ([T][768], which also holds the patch rows):
    // 0.74 M floats at vit_tiny's 311 tokens, below the 2.36 M an OSNet_x1_0 chunk takes per crop
    const size_t T = v.tokens;
    Workspace ws;
    ws.blob = (size_t)m->in_h * m->in_w * 3;
    ws.bufA = ws.bufB = ws.Y[0][0] = T * D;
    ws.x1 = std::max(T * 3 * D, (size_t)vits::MAX_FEAT);
    ws.Y[0][1] = T * vits::MLP;
    return ws;
}

// ---- CSPReID-n (reid/backbones/cspreid_n.py): stem, four C3k2 stages, SPPF, LightSelfAttention, three BNNeck3 ----
// The C3k2 shapes (in, out, bottlenecks) of stages 1-4
static const int kCspStage[4][3] = {{64, 128, 1}, {128, 256, 1}, {256, 384, 2}, {384, 512, 1}};
Workspace layout_cspreid(ReidModel* m, BlobCursor& take, WgmmaPack& pack) {
    CspW& cs = m->cs;
    m->stem_w = take((size_t)27 * csp::STEM_C);
    m->stem_b = take(csp::STEM_C);
    int i = 0;
    auto conv = [&](int K, int N) {
        RnConv& c = cs.conv[i++];
        const size_t w = take((size_t)K * N);
        c.b = take(N);
        pack.add(c.w, w, K, N);
    };
    conv(9 * csp::STEM_C, 64);
    for (int s = 0; s < 4; ++s) {
        const int cin = kCspStage[s][0], cout = kCspStage[s][1], n = kCspStage[s][2], mid = cout / 2;
        conv(cin, 2 * mid);
        for (int b = 0; b < n; ++b) {
            conv(mid, mid / 2);
            conv(9 * (mid / 2), mid);
        }
        conv((2 + n) * mid, cout);
        if (s < 3) conv(9 * cout, cout);
    }
    conv(csp::C, csp::SPPF_C);
    conv(4 * csp::SPPF_C, csp::C);
    const size_t attn[5] = {(size_t)csp::C * csp::HID, (size_t)csp::HID * csp::C, 9 * (size_t)csp::C, csp::C, csp::C};
    for (int k = 0; k < 5; ++k) cs.attn[k] = take(attn[k]);
    for (int h = 0; h < 3; ++h) {
        cs.head[2 * h] = take((size_t)csp::C * csp::C);
        cs.head[2 * h + 1] = take(csp::C);
    }
    // per crop (at H x W = 256 x 128; twice as much at 256 x 256): the crop; two maps as large as the first stem conv's
    // output (H/2 x W/2 x 32, also stage 1's C3k2 output H/4 x W/4 x 128); stage 1's C3k2 concatenation
    // (H/4 x W/4 x 192, the largest); a bottleneck's hidden map (H/4 x W/4 x 32); the head row: 1.1 M floats (2.2 M at
    // 256 x 256), below the 2.36 M an OSNet_x1_0 chunk takes per crop, so the chunk keeps its size.
    const size_t px = (size_t)(m->in_h / 4) * (m->in_w / 4);
    Workspace ws;
    ws.blob = (size_t)m->in_h * m->in_w * 3;
    ws.bufA = ws.bufB = std::max((size_t)(m->in_h / 2) * (m->in_w / 2) * csp::STEM_C, px * 128);
    ws.x1 = px * 192;
    ws.Y[0][0] = px * 32;
    ws.sums[0] = csp::FEAT;
    return ws;
}

// The A/B kernel switches of the OSNet family, and for OSNet (arch 1) the tensor-core copies of every 1x1 weight that
// fits the tensor-core kernel's accumulators and shared memory
void setup_osnet_kernels(ReidModel* m, const float* host) {
    const char* env = getenv("BOXMOT_B200_REID_TC");
    // At OSNet_x0_25's K,N <= 128 every 1x1 layer is bandwidth-bound, and on an H100 this unpipelined kernel is
    // 1.1-2.4x slower than the float32 CUDA-core GEMM (tests/test_gpu_pointwise_tc.py prints both), so the
    // standalone tensor-core GEMM is opt-in.
    m->use_tc = env && env[0] == '1' && m->arch == ARCH_OSNET;   // LMBN_n runs the float32 CUDA-core kernels only
    const char* lv = getenv("BOXMOT_B200_LIGHT_V1");
    m->light_v2 = !(lv && lv[0] == '1');
    if (const char* cv = getenv("BOXMOT_B200_LIGHT_CHAIN")) m->light_chain = !(cv[0] == '0');
    if (const char* cv = getenv("BOXMOT_B200_LIGHT_TC")) m->light_tc = cv[0] == '1';
    if (const char* cv = getenv("BOXMOT_B200_LIGHT_SMALL")) m->light_small = cv[0] == '1';
    if (const char* cv = getenv("BOXMOT_B200_CHAIN_VAR")) m->chain_var = atoi(cv);
    const char* pv = getenv("BOXMOT_B200_PW_V1");
    m->pw_v2 = !(pv && pv[0] == '1');
    if (const char* cv = getenv("BOXMOT_B200_PW_SMALL")) m->pw_small = !(cv[0] == '0');
    if (m->arch != ARCH_OSNET) return;
    std::vector<float> packed;
    struct Todo { TcW* dst; size_t w; int K, N; size_t at; };
    std::vector<Todo> todo;
    auto add = [&](TcW* dst, size_t w, int K, int N) {
        const int Kpad = (K + 7) / 8 * 8, Npad = (N + 15) / 16 * 16;
        if (Npad > tc::NPAD_MAX || tc::smem_bytes(Kpad, Npad) > 200 * 1024) return;
        dst->Kpad = Kpad; dst->Npad = Npad;
        todo.push_back({dst, w, K, N, packed.size()});
        packed.resize(packed.size() + 2 * (size_t)Npad * Kpad);
    };
    for (BlockW& b : m->blocks) {
        add(&b.tc_c1, b.c1w, b.cin, b.mid);
        add(&b.tc_c, b.cw, b.mid + (b.has_ds ? b.cin : 0), b.cout);
        if (b.mid % 16 == 0)
            for (int l = 0; l < 10; ++l) add(&b.light_tc[l], b.light[l].pw, b.mid, b.mid);
    }
    for (int s = 0; s < 2; ++s) add(&m->tc_trans[s], m->trans_w[s], m->c[s + 1], m->c[s + 1]);
    add(&m->tc_c5, m->c5w, m->c[3], m->c[3]);
    for (auto& t : todo) tc::pack_weights(host + t.w, t.K, t.N, t.dst->Kpad, t.dst->Npad, packed.data() + t.at);
    if (!packed.empty()) {
        RCUDA_OK(cudaMalloc(&m->d_wtc, sizeof(float) * packed.size()));
        RCUDA_OK(cudaMemcpy(m->d_wtc, packed.data(), sizeof(float) * packed.size(), cudaMemcpyHostToDevice));
        for (auto& t : todo) t.dst->w = m->d_wtc + t.at;
    }
}
}  // namespace

ReidModel* reid_load(const char* path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error(std::string("cannot open ReID blob: ") + path);
    int32_t hdr[16];
    f.read(reinterpret_cast<char*>(hdr), sizeof(hdr));
    if (!f || (uint32_t)hdr[0] != BLOB_MAGIC || hdr[1] != 1 || hdr[2] < ARCH_OSNET || hdr[2] > ARCH_CSPREID)
        throw std::runtime_error("not a version-1 .b200reid blob (export it with boxmot_b200.weights.export_blob)");
    ReidModel* m = new ReidModel();
    try {
        read_header(m, hdr);
        std::vector<int32_t> table;   // MobileNetV2's block table sits between the header and the payload
        if (m->arch == ARCH_MOBILENETV2) {
            table.resize((size_t)hdr[4] * 4);
            f.read(reinterpret_cast<char*>(table.data()), sizeof(int32_t) * table.size());
        }
        const size_t n_floats = (size_t)hdr[8];
        std::vector<float> host(n_floats);
        f.read(reinterpret_cast<char*>(host.data()), sizeof(float) * n_floats);
        if (!f) throw std::runtime_error("truncated ReID blob");
        BlobCursor take;
        WgmmaPack pack;
        Workspace ws;
        switch (m->arch) {
            case ARCH_MOBILENETV2: ws = layout_mobilenetv2(m, table, take); break;
            case ARCH_RESNET: ws = layout_resnet(m, hdr, take, pack); break;
            case ARCH_CLIP: ws = layout_clip(m, take, pack); break;
            case ARCH_MLFN: ws = layout_mlfn(m, take, pack); break;
            case ARCH_HACNN: ws = layout_hacnn(m, take, pack); break;
            case ARCH_VIT: ws = layout_vits(m, take, pack); break;
            case ARCH_CSPREID: ws = layout_cspreid(m, take, pack); break;
            default: ws = layout_osnet(m, hdr, take); break;
        }
        if (take.o != n_floats) throw std::runtime_error("ReID blob size does not match its header");

        RCUDA_OK(cudaMalloc(&m->d_w, sizeof(float) * n_floats));
        RCUDA_OK(cudaMemcpy(m->d_w, host.data(), sizeof(float) * n_floats, cudaMemcpyHostToDevice));
        if (!pack.todo.empty()) {
            std::vector<float> packed(pack.n);
            for (auto& t : pack.todo) rn::pack_conv_weights(host.data() + t.w, t.K, t.N, packed.data() + t.at);
            RCUDA_OK(cudaMalloc(&m->d_wrn, sizeof(float) * pack.n));
            RCUDA_OK(cudaMemcpy(m->d_wrn, packed.data(), sizeof(float) * pack.n, cudaMemcpyHostToDevice));
            for (auto& t : pack.todo) *t.dst = m->d_wrn + t.at;
        }
        const bool osnet_family = m->arch == ARCH_OSNET || m->arch == ARCH_LMBN_N || m->arch == ARCH_OSNET_IN;
        if (osnet_family) setup_osnet_kernels(m, host.data());

        // workspace for one chunk of crops
        if (const char* ce = getenv("BOXMOT_B200_REID_CHUNK")) {
            const int v = atoi(ce);
            if (v >= 8 && v <= 1024) m->chunk = v;
        }
        // LMBN_n's maps are 1.5x taller and it keeps the trunk output: fewer crops per chunk, so that a chunk's
        // workspace stays within what an OSNet of the same widths at 256x128 takes for the configured chunk
        if (m->arch == ARCH_LMBN_N)
            m->chunk = std::max(8, (int)((size_t)m->chunk * osnet_workspace(m, IN_H, false).total() / ws.total()));
        const size_t CH = m->chunk;
        auto alloc = [&](float*& p, size_t per_crop) {
            if (per_crop) RCUDA_OK(cudaMalloc(&p, sizeof(float) * CH * per_crop));
        };
        alloc(m->blob, ws.blob);
        alloc(m->bufA, ws.bufA);
        alloc(m->bufB, ws.bufB);
        alloc(m->x1, ws.x1);
        for (int b = 0; b < 4; ++b) {
            for (int k = 0; k < 2; ++k) alloc(m->Y[b][k], ws.Y[b][k]);
            alloc(m->sums[b], ws.sums[b]);
        }
        alloc(m->gates, ws.gates);
        alloc(m->in_tmp, ws.in_tmp);
        alloc(m->trunk, ws.trunk);
        alloc(m->pooled, ws.pooled);
        if (m->arch == ARCH_HACNN) RCUDA_OK(cudaMalloc(&m->d_n4, sizeof(int)));
        // tensor-core path: the default wherever its kernel instances cover the widths (BOXMOT_B200_REID_FP32=1
        // keeps the float32 CUDA-core kernels of round 1, e.g. for A/B runs)
        if (osnet_family) {
            const char* fe = getenv("BOXMOT_B200_REID_FP32");
            if (!(fe && fe[0] == '1') && tcx::plan_supported(m)) m->tc = tcx::plan_build(m, host.data());
        }
    } catch (...) {
        reid_free(m);
        throw;
    }
    return m;
}

void reid_free(ReidModel* m) {
    if (!m) return;
    cudaFree(m->d_w); cudaFree(m->d_wtc); cudaFree(m->blob); cudaFree(m->bufA); cudaFree(m->bufB); cudaFree(m->x1);
    for (int b = 0; b < 4; ++b) { cudaFree(m->Y[b][0]); cudaFree(m->Y[b][1]); cudaFree(m->sums[b]); }
    cudaFree(m->gates); cudaFree(m->trunk); cudaFree(m->pooled); cudaFree(m->in_tmp); cudaFree(m->d_wrn);
    cudaFree(m->d_n4);
    tcx::plan_free(m->tc);
    delete m;
}

int reid_feature_dim(const ReidModel* m) { return m->feat; }
void reid_set_preprocess(ReidModel* m, int mode) { m->preprocess = mode ? 1 : 0; }
const float* reid_last_input_blob(const ReidModel* m) { return m->blob; }
void reid_set_profile(ReidModel* m, bool on) { m->profile = on; }
// Fold the events recorded since the last call into per-class totals (the stream must be idle).
void reid_profile_collect(ReidModel* m, double* ms, int* launches) {
    for (size_t i = 0; i < m->prof_cls.size(); ++i) {
        float t = 0.f;
        cudaEventElapsedTime(&t, m->prof_ev[2 * i], m->prof_ev[2 * i + 1]);
        m->prof_ms[m->prof_cls[i]] += t;
        m->prof_launches[m->prof_cls[i]] += 1;
        cudaEventDestroy(m->prof_ev[2 * i]);
        cudaEventDestroy(m->prof_ev[2 * i + 1]);
    }
    m->prof_ev.clear();
    m->prof_cls.clear();
    for (int c = 0; c < REID_N_CLASSES; ++c) {
        if (ms) ms[c] = m->prof_ms[c];
        if (launches) launches[c] = m->prof_launches[c];
        m->prof_ms[c] = 0;
        m->prof_launches[c] = 0;
    }
}
void reid_set_debug_stop(ReidModel* m, int stage) { m->debug_stop = stage; }
const float* reid_debug_tensor(const ReidModel* m, size_t* floats_per_crop) {
    if (floats_per_crop) *floats_per_crop = m->debug_floats_per_crop;
    return m->debug_ptr;
}

namespace {
struct Launcher {
    ReidModel* m;
    const int* d_n;
    int off, cap, upper;  // upper = host-side bound on crops in this chunk (grid sizing)
    cudaStream_t st;
    int launches = 0;
    // the kernel instance of the last pointwise / LightConv launch (standalone entry points report it):
    // pointwise {BN, threads, gated, 0}; LightConv {kind, C, W, R} with kind 1 k_lightconv, 2 k_lightconv2,
    // 3 k_lightchain (R = chain tile rows)
    int inst[4] = {0, 0, 0, 0};

    void begin(int cls) {
        if (!m->profile) return;
        cudaEvent_t e0, e1;
        RCUDA_OK(cudaEventCreate(&e0));
        RCUDA_OK(cudaEventCreate(&e1));
        m->prof_ev.push_back(e0);
        m->prof_ev.push_back(e1);
        m->prof_cls.push_back(cls);
        RCUDA_OK(cudaEventRecord(e0, st));
    }
    // counts every launch, so that reid_forward's count and the profile's per-class counts agree
    void end() {
        ++launches;
        if (!m->profile) return;
        RCUDA_OK(cudaEventRecord(m->prof_ev.back(), st));
    }

    void pointwise_tc(const PwArgs& a) {
        tc::Args t{};
        t.in = a.in;
        for (int b = 0; b < 4; ++b) t.branch[b] = a.branch[b];
        t.gates = a.gates; t.w_tc = a.w_tc; t.bias = a.bias; t.residual = a.residual; t.out = a.out;
        t.K = a.K; t.N = a.N; t.Kpad = a.Kpad; t.Npad = a.Npad; t.mid = a.mid; t.HW = a.HW; t.relu = a.relu;
        const size_t smem = tc::smem_bytes(a.Kpad, a.Npad);
        int per_sm = (int)((220 * 1024) / (smem + 1024));
        per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
        const int tiles = (int)(((size_t)upper * a.HW) / tc::TILE_M);
        const int grid = tiles < m->sms * per_sm ? tiles : m->sms * per_sm;
        begin(CLS_POINTWISE);
        if (a.gates) {
            RCUDA_OK(cudaFuncSetAttribute(tc::k_pointwise_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            tc::k_pointwise_tc<true><<<grid, tc::THREADS, smem, st>>>(t, d_n, off, cap);
        } else {
            RCUDA_OK(cudaFuncSetAttribute(tc::k_pointwise_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            tc::k_pointwise_tc<false><<<grid, tc::THREADS, smem, st>>>(t, d_n, off, cap);
        }
        end();
    }
    void pointwise(const PwArgs& a) {
        if (m->use_tc && a.w_tc && a.HW % tc::TILE_M == 0) { pointwise_tc(a); return; }
        const int N = a.N;
        const size_t Mmax = (size_t)upper * a.HW;
        if (N % 64 == 0) launch_pw<64>(a, Mmax);
        else if (N % 32 == 0 || N > 16) launch_pw<32>(a, Mmax);
        else launch_pw<16>(a, Mmax);
    }
    template <int BN>
    void launch_pw(const PwArgs& a, size_t Mmax) {
        constexpr int BM = (256 / (BN / 4)) * 8;
        dim3 grid((unsigned)((Mmax + BM - 1) / BM), (unsigned)((a.N + BN - 1) / BN));
        if (m->pw_v2 && m->pw_small) {   // 128-thread CTAs: half the rows per CTA, twice the CTAs (A/B switch)
            constexpr int BMs = (128 / (BN / 4)) * 8;
            constexpr size_t smem = 2 * sizeof(float4) * (4 * (BMs + 2) + 16 * BN / 4);
            dim3 g((unsigned)((Mmax + BMs - 1) / BMs), (unsigned)((a.N + BN - 1) / BN));
            begin(CLS_POINTWISE);
            inst[0] = BN; inst[1] = 128; inst[2] = a.gates != nullptr; inst[3] = 0;
            if (a.gates) k_pointwise2<BN, true, 128><<<g, 128, smem, st>>>(a, d_n, off, cap);
            else k_pointwise2<BN, false, 128><<<g, 128, smem, st>>>(a, d_n, off, cap);
            end();
            return;
        }
        inst[0] = BN; inst[1] = 256; inst[2] = a.gates != nullptr; inst[3] = 0;
        if (m->pw_v2) {
            constexpr size_t smem = 2 * sizeof(float4) * (4 * (BM + 2) + 16 * BN / 4);
            begin(CLS_POINTWISE);
            if (a.gates) {
                if (smem > 48 * 1024)
                    RCUDA_OK(cudaFuncSetAttribute(k_pointwise2<BN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                k_pointwise2<BN, true><<<grid, 256, smem, st>>>(a, d_n, off, cap);
            } else {
                if (smem > 48 * 1024)
                    RCUDA_OK(cudaFuncSetAttribute(k_pointwise2<BN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                k_pointwise2<BN, false><<<grid, 256, smem, st>>>(a, d_n, off, cap);
            }
            end();
            return;
        }
        begin(CLS_POINTWISE);
        if (a.gates) k_pointwise<BN, true><<<grid, 256, 0, st>>>(a, d_n, off, cap);
        else k_pointwise<BN, false><<<grid, 256, 0, st>>>(a, d_n, off, cap);
        end();
    }
    template <int C, int W, int R, int PPL = 4, int MINB = 2, bool TC = false, int NT = 256>
    void launch_light2(const LightArgs& a, int n_branches) {
        const int tiles = (a.H + R - 1) / R;
        const size_t smem = light2_smem_bytes((R + 2) * (W + 2), C, NT, PPL, TC);
        if (smem > 48 * 1024)
            RCUDA_OK(cudaFuncSetAttribute(k_lightconv2<C, W, R, PPL, MINB, TC, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        begin(CLS_LIGHTCONV);
        inst[0] = 2; inst[1] = C; inst[2] = W; inst[3] = R;
        k_lightconv2<C, W, R, PPL, MINB, TC, NT><<<dim3(tiles, n_branches, upper), NT, smem, st>>>(a, d_n, off, cap);
        end();
    }
    template <int C, int W, int R, int NT>
    void launch_chain(const ChainArgs& a) {
        const int tiles = a.H / R;
        constexpr size_t smem = chain_smem_bytes<C, W, R, NT>();
        RCUDA_OK(cudaFuncSetAttribute(k_lightchain<C, W, R, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        begin(CLS_LIGHTCONV);
        inst[0] = 3; inst[1] = C; inst[2] = W; inst[3] = R;
        k_lightchain<C, W, R, NT><<<dim3(tiles, 4, upper), NT, smem, st>>>(a, d_n, off, cap);
        end();
    }
    // whole-branch LightConv chains for the osnet_x0_25 stage shapes; returns the tile rows used (0 = not covered)
    int light_chain(const ChainArgs& a, int C, int W) {
        if (C == 16 && W == 32) {
            if (m->chain_var == 2) return 0;   // stage 2 per level (8-row chain tiles recompute 25 % halo rows)
            if (m->chain_var == 1) { launch_chain<16, 32, 16, 512>(a); return 16; }
            launch_chain<16, 32, 8, 256>(a); return 8;
        }
        if (C == 24 && W == 16) { launch_chain<24, 16, 16, 256>(a); return 16; }
        if (C == 32 && W == 8) { launch_chain<32, 8, 16, 256>(a); return 16; }
        return 0;
    }
    // shape-specialised LightConv (the three OSBlock stages of osnet_x0_25 and osnet_x1_0); false = not covered
    bool light2(const LightArgs& a, int n_branches) {
#define BMB_LIGHT2(CC, WW, RR) \
        if (a.C == CC && a.W == WW && a.R == RR) { launch_light2<CC, WW, RR>(a, n_branches); return true; }
        if (m->light_small && a.C == 16 && a.W == 32 && a.R == 8) {   // four 128-thread CTAs per SM (A/B switch)
            launch_light2<16, 32, 8, 2, 4, false, 128>(a, n_branches);
            return true;
        }
        if (m->light_tc && a.C == 16 && a.W == 32 && a.R == 16 && a.wtc[0]) {   // tensor-core 1x1 stage (opt-in)
            launch_light2<16, 32, 16, 4, 2, true>(a, n_branches);
            return true;
        }
        BMB_LIGHT2(16, 32, 16) BMB_LIGHT2(24, 16, 16) BMB_LIGHT2(32, 8, 16)
        BMB_LIGHT2(64, 32, 8) BMB_LIGHT2(96, 16, 4) BMB_LIGHT2(128, 8, 8)
#undef BMB_LIGHT2
        return false;
    }
    // instance norm (arch 4): statistics of x [crops][HW][C] into stats, timed under `cls`
    void in_stats(const float* x, int HW, int C, double2* stats, int cls) {
        begin(cls);
        k_in_stats<<<dim3((C + INS_LANES - 1) / INS_LANES, upper), INS_LANES * INS_STRIPES, 0, st>>>(x, HW, C, d_n, off,
                                                                                                       cap, stats);
        end();
    }
    void in_apply(const float* x, const float* residual, float* out, int HW, int C, const float* gamma,
                  const float* beta, const double2* stats, int relu, int cls) {
        begin(cls);
        k_in_apply<<<m->sms * 8, 256, 0, st>>>(x, residual, out, HW, C, gamma, beta, stats, relu, d_n, off, cap);
        end();
    }
    // one ResNet convolution (rn::k_conv_tc) over the output pixels of at most `upper` crops
    void conv_tc(const rn::ConvArgs& a) {
        const int BN = rn::tile_n(a.N);
        const dim3 grid((unsigned)(((size_t)upper * a.Ho * a.Wo + rn::BM - 1) / rn::BM), (unsigned)(a.N / BN));
        begin(a.k0 == 3 ? CLS_LIGHTCONV : CLS_POINTWISE);
        if (a.out_ld) {   // a stream's channel slice of a concatenated map (HACNN)
            if (BN == 128) conv_tc_slice<128>(a, grid);
            else if (BN == 64) conv_tc_slice<64>(a, grid);
            else conv_tc_slice<32>(a, grid);
        } else if (a.relu == 4) {   // exact GELU: the ViT-Nano / ViT-Tiny MLP's fc1
            if (BN == 128) conv_tc_gelu<128>(a, grid);
            else conv_tc_gelu<64>(a, grid);
        } else if (a.relu == 3) {   // relu(residual + relu(acc + bias)): MLFN's fm_conv3
            if (BN == 128) {
                RCUDA_OK(cudaFuncSetAttribute(rn::k_conv_tc<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<128>()));
                rn::k_conv_tc<128, true><<<grid, rn::THREADS, rn::smem_bytes<128>(), st>>>(a, d_n, off, cap);
            } else {
                RCUDA_OK(cudaFuncSetAttribute(rn::k_conv_tc<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<64>()));
                rn::k_conv_tc<64, true><<<grid, rn::THREADS, rn::smem_bytes<64>(), st>>>(a, d_n, off, cap);
            }
        } else if (BN == 128) {
            RCUDA_OK(cudaFuncSetAttribute(rn::k_conv_tc<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<128>()));
            rn::k_conv_tc<128><<<grid, rn::THREADS, rn::smem_bytes<128>(), st>>>(a, d_n, off, cap);
        } else {
            RCUDA_OK(cudaFuncSetAttribute(rn::k_conv_tc<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<64>()));
            rn::k_conv_tc<64><<<grid, rn::THREADS, rn::smem_bytes<64>(), st>>>(a, d_n, off, cap);
        }
        end();
    }
    // one ConvBNSiLU on k_conv_tc's SILU instances (CSPReID-n): a.relu 5 SiLU, 6 residual + SiLU; pitches in a.in_ld,
    // a.res_ld, a.out_ld
    void conv_tc_silu(const rn::ConvArgs& a) {
        const int BN = rn::tile_n(a.N);
        const dim3 grid((unsigned)(((size_t)upper * a.Ho * a.Wo + rn::BM - 1) / rn::BM), (unsigned)(a.N / BN));
        begin(a.k0 == 3 ? CLS_LIGHTCONV : CLS_POINTWISE);
        if (a.relu == 6) {
            if (BN == 128) launch_silu<128, 2>(a, grid);
            else if (BN == 64) launch_silu<64, 2>(a, grid);
            else launch_silu<32, 2>(a, grid);
        } else {
            if (BN == 128) launch_silu<128, 1>(a, grid);
            else if (BN == 64) launch_silu<64, 1>(a, grid);
            else launch_silu<32, 1>(a, grid);
        }
        end();
    }
    template <int BN, int SILU>
    void launch_silu(const rn::ConvArgs& a, dim3 grid) {
        auto k = rn::k_conv_tc<BN, false, false, false, SILU>;
        RCUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<BN>()));
        k<<<grid, rn::THREADS, rn::smem_bytes<BN>(), st>>>(a, d_n, off, cap);
    }
    // CSPReID-n: the 3 -> 32 3x3 stride-2 stem of the H x Wd crop, timed under `stem`
    void csp_stem(const float* blob, int H, int Wd, const float* w, const float* b, float* out) {
        begin(CLS_STEM);
        csp::k_stem<<<m->sms * 8, 256, 0, st>>>(blob, H, Wd, w, b, d_n, off, cap, out);
        end();
    }
    // CSPReID-n: SPPF's three chained 3x3 max pools of slice 0 of buf [crops][H][Wd][4 c] into slices 1-3
    void csp_sppf(float* buf, int H, int Wd, int c) {
        begin(CLS_MAXPOOL);
        csp::k_sppf<<<m->sms * 8, 256, 0, st>>>(buf, H, Wd, c, d_n, off, cap);
        end();
    }
    // CSPReID-n: LightSelfAttention of x [crops][H][Wd][512] into out; p = fc.0, fc.2, dw, dw shift, spatial 1x1
    void csp_attn(const float* x, int H, int Wd, const float* const* p, float* out) {
        begin(CLS_GATES);
        csp::k_attn<<<upper, csp::C, 0, st>>>(x, H, Wd, p[0], p[1], p[2], p[3], p[4], d_n, off, cap, out);
        end();
    }
    // CSPReID-n: pools, three BNNeck3 GEMVs, interleave and L2 norm of x [crops][H][Wd][512] into the caller's rows;
    // p = W, b of bn_global, bn_part0, bn_part1; raw (optional) gets the rows before the norm
    void csp_head(const float* x, int H, int Wd, const float* const* p, const CropDesc* crops, float* out, int out_ld,
                  float* raw) {
        begin(CLS_HEAD);
        csp::k_head<<<(upper + csp::HEAD_CROPS - 1) / csp::HEAD_CROPS, csp::C, 0, st>>>(
            x, H, Wd, p[0], p[1], p[2], p[3], p[4], p[5], crops, d_n, off, cap, out, out_ld, raw);
        end();
    }
    template <int BN>
    void conv_tc_gelu(const rn::ConvArgs& a, dim3 grid) {
        RCUDA_OK(cudaFuncSetAttribute(rn::k_conv_tc<BN, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<BN>()));
        rn::k_conv_tc<BN, false, false, true><<<grid, rn::THREADS, rn::smem_bytes<BN>(), st>>>(a, d_n, off, cap);
    }
    template <int BN>
    void conv_tc_slice(const rn::ConvArgs& a, dim3 grid) {
        RCUDA_OK(cudaFuncSetAttribute(rn::k_conv_tc<BN, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rn::smem_bytes<BN>()));
        rn::k_conv_tc<BN, false, true><<<grid, rn::THREADS, rn::smem_bytes<BN>(), st>>>(a, d_n, off, cap);
    }
    // HACNN: the 3x3 stride-2 stem of the 160x64 crop, timed under `stem`
    void hacnn_stem(const float* blob, const float* w, const float* b, float* out) {
        begin(CLS_STEM);
        hacnn::k_stem<<<m->sms * 8, 256, 0, st>>>(blob, w, b, d_n, off, cap, out);
        end();
    }
    // HACNN: 3x3 pad-1 pool of x [imgs][H][Wd][C], the max at stride 2 or the average (/ 9) at stride 1
    void hacnn_pool(bool max, const float* x, int H, int Wd, int C, float* out) {
        begin(max ? CLS_MAXPOOL : CLS_AVGPOOL);
        if (max) hacnn::k_pool3<true><<<m->sms * 8, 256, 0, st>>>(x, H, Wd, C, 2, d_n, off, cap, out);
        else hacnn::k_pool3<false><<<m->sms * 8, 256, 0, st>>>(x, H, Wd, C, 1, d_n, off, cap, out);
        end();
    }
    // HACNN: the soft attention's s and v and the hard attention's theta of x [crops][H][Wd][C], timed under `gates`
    void hacnn_attn(const float* x, int H, int Wd, int C, const hacnn::AttnW& a, int level, float* s, float* v,
                    float* theta) {
        begin(CLS_GATES);
        hacnn::k_attn<<<upper, 256, 0, st>>>(x, H, Wd, C, a, level, d_n, off, cap, s, v, theta);
        end();
    }
    void hacnn_attn_apply(float* x, int HW, int C, const float* s, const float* v, const float* b) {
        begin(CLS_GATES);
        hacnn::k_attn_apply<<<m->sms * 8, 256, 0, st>>>(x, HW, C, s, v, b, d_n, off, cap);
        end();
    }
    // HACNN: the four regions' STN samples of src, resized to h x w (+ prev) into [crops][4][h][w][C], under `gates`
    void hacnn_stn(const float* src, int H, int Wd, int C, const float* theta, const float* prev, int h, int w,
                   float* out) {
        begin(CLS_GATES);
        hacnn::k_stn<<<m->sms * 8, 256, 0, st>>>(src, H, Wd, C, theta, prev, h, w, d_n, off, cap, out);
        end();
    }
    void hacnn_head_pool(const float* x3, int HW3, const float* loc, int HWl, float* pg, float* pl) {
        begin(CLS_HEAD);
        hacnn::k_head_pool<<<upper, 256, 0, st>>>(x3, HW3, loc, HWl, d_n, off, cap, pg, pl);
        end();
    }
    void hacnn_head(const float* v, const CropDesc* crops, float* out, int out_ld) {
        begin(CLS_HEAD);
        hacnn::k_head<<<upper, 256, 0, st>>>(v, crops, d_n, off, cap, out, out_ld);
        end();
    }
    // MLFN: grouped 3x3 (+ bias, ReLU, gate) of x [crops][H][Wd][C], group width gw, timed under `lightconv`
    void group_conv(const float* x, int H, int Wd, int C, int gw, int stride, const float* w, const float* bias,
                    const float* gates, float* out) {
        const int Ho = (H - 1) / stride + 1, Wo = (Wd - 1) / stride + 1;
        const size_t items = (size_t)upper * Ho * (Wo / 4) * (C / 4);
        const unsigned grid = (unsigned)((items + 255) / 256);
        begin(CLS_LIGHTCONV);
        switch (gw) {
            case 4: mlfn::k_group_conv<4><<<grid, 256, 0, st>>>(x, H, Wd, C, stride, w, bias, gates, mlfn::SHAT, d_n, off, cap, out); break;
            case 8: mlfn::k_group_conv<8><<<grid, 256, 0, st>>>(x, H, Wd, C, stride, w, bias, gates, mlfn::SHAT, d_n, off, cap, out); break;
            case 16: mlfn::k_group_conv<16><<<grid, 256, 0, st>>>(x, H, Wd, C, stride, w, bias, gates, mlfn::SHAT, d_n, off, cap, out); break;
            case 32: mlfn::k_group_conv<32><<<grid, 256, 0, st>>>(x, H, Wd, C, stride, w, bias, gates, mlfn::SHAT, d_n, off, cap, out); break;
            default: throw std::runtime_error("MLFN grouped convolution: group width must be 4, 8, 16 or 32");
        }
        end();
    }
    // MLFN: average pool of x [crops][HW][C] into rows [crops][C], timed under `gates`
    void mlfn_gap(const float* x, int HW, int C, float* out) {
        begin(CLS_GATES);
        mlfn::k_mlfn_gap<<<dim3(C / 64, upper), 256, 0, st>>>(x, HW, C, d_n, off, cap, out);
        end();
    }
    // MLFN: the FSM's last layer + sigmoid into columns col .. col + 31 of s_hat, timed under `gates`
    void mlfn_gate(const float* h, int F1, const float* w, const float* b, float* s_hat, int col) {
        begin(CLS_GATES);
        mlfn::k_mlfn_gate<<<(upper + 7) / 8, 256, 0, st>>>(h, F1, w, b, d_n, off, cap, s_hat, col);
        end();
    }
    // CLIP: LayerNorm of T token rows per crop (EMBED: token assembly + ln_pre), timed under `gates`
    void vit_layernorm(bool embed, const float* in, const float* pos, const float* g, const float* b, int T, float* out) {
        const int grid = (int)std::min<size_t>(((size_t)upper * T + 7) / 8, (size_t)m->sms * 16);
        begin(CLS_GATES);
        if (embed) vit::k_vit_layernorm<true><<<grid, 256, 0, st>>>(in, pos, g, b, T, d_n, off, cap, out);
        else vit::k_vit_layernorm<false><<<grid, 256, 0, st>>>(in, pos, g, b, T, d_n, off, cap, out);
        end();
    }
    // CLIP (width 768) and ViT-Nano / ViT-Tiny (width 192): multi-head attention of every (crop, head, query block),
    // timed under `lightconv`
    void vit_attention(const float* qkv, int T, float* out, int width = vit::D) {
        const size_t smem = vit::attention_smem_bytes(T);
        const dim3 grid((T + vit::ATT_QB - 1) / vit::ATT_QB, width / vit::HD, upper);
        begin(CLS_LIGHTCONV);
        if (width == vit::D) {
            RCUDA_OK(cudaFuncSetAttribute(vit::k_vit_attention<vit::D, vit::MAX_T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            vit::k_vit_attention<vit::D, vit::MAX_T><<<grid, vit::ATT_THREADS, smem, st>>>(qkv, T, d_n, off, cap, out);
        } else {
            RCUDA_OK(cudaFuncSetAttribute(vit::k_vit_attention<vits::D, vits::MAX_T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            vit::k_vit_attention<vits::D, vits::MAX_T><<<grid, vit::ATT_THREADS, smem, st>>>(qkv, T, d_n, off, cap, out);
        }
        end();
    }
    // ViT-Nano / ViT-Tiny: LayerNorm of T 192-wide rows per crop, timed under `gates`
    void vits_layernorm(const float* in, const float* g, const float* b, int T, float* out) {
        const int grid = (int)std::min<size_t>(((size_t)upper * T + 7) / 8, (size_t)m->sms * 16);
        begin(CLS_GATES);
        vits::k_vits_layernorm<<<grid, 256, 0, st>>>(in, g, b, T, d_n, off, cap, out);
        end();
    }
    // ViT-Nano AIN blocks: AdaptiveINLN of every crop (one CTA each), timed under `gates`
    void vits_ain(const float* in, const float* a, const float* b, const float* s, int T, float* out) {
        const size_t smem = vits::ain_smem_bytes(T);
        RCUDA_OK(cudaFuncSetAttribute(vits::k_vits_ain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        begin(CLS_GATES);
        vits::k_vits_ain<<<upper, vits::AIN_THREADS, smem, st>>>(in, T, a, b, s, d_n, off, cap, out);
        end();
    }
    // ViT-Nano / ViT-Tiny head (pooling, projections, BNNecks, L2 norm or the un-normalised tap), timed under `head`
    void vits_head(const float* x, int T, int gh, int gw, int pool, int proj, const float* hw, const CropDesc* crops,
                   float* out, int out_ld, float* tap) {
        begin(CLS_HEAD);
        vits::k_vits_head<<<upper, vits::HEAD_THREADS, 0, st>>>(x, T, gh, gw, pool, proj, hw, crops, d_n, off, cap, out,
                                                                out_ld, tap);
        end();
    }
    // ChannelGate of an OSBlock: one CTA per crop
    void gates(const GateArgs& a) {
        begin(CLS_GATES);
        k_gates<<<upper, 128, sizeof(float) * (4 * a.C + 4 * a.hid), st>>>(a, d_n, off, cap);
        end();
    }
    // head of OSNet (fc + ReLU) and of ResNet / MobileNetV2 (wfc null: the pooled map is the embedding), L2-normalised
    // into the caller's rows
    void head(const float* x, int HW, int C, const float* wfc, const float* bfc, int feat, const CropDesc* crops,
              float* out, int out_ld) {
        const int groups = 256 / C > 0 ? 256 / C : 1;
        begin(CLS_HEAD);
        k_head<<<upper, 256, sizeof(float) * (C + 32 + (size_t)groups * C), st>>>(x, HW, C, wfc, bfc, feat, crops, d_n,
                                                                                   off, cap, out, out_ld);
        end();
    }
    // 7x7 stride-2 stem of the OSNet family (raw: the instance-norm stem's bare convolution)
    void stem(bool raw, const float* blob, const float* w, const float* bias, int C0, float* out, int in_h) {
        const size_t smem = sizeof(float) * ((size_t)((ST_IR * ST_IC * 3 + 3) & ~3) + 147 * 16);
        const dim3 grid(in_h / 2 / ST_R, upper);
        begin(CLS_STEM);
        if (raw) {
            RCUDA_OK(cudaFuncSetAttribute(k_stem<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k_stem<true><<<grid, 256, smem, st>>>(blob, w, nullptr, C0, d_n, off, cap, out, in_h);
        } else {
            RCUDA_OK(cudaFuncSetAttribute(k_stem<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k_stem<false><<<grid, 256, smem, st>>>(blob, w, bias, C0, d_n, off, cap, out, in_h);
        }
        end();
    }
    void maxpool(const float* in, int H, int W, int C, float* out) {
        begin(CLS_MAXPOOL);
        k_maxpool3s2<<<m->sms * 8, 256, 0, st>>>(in, H, W, C, d_n, off, cap, out);
        end();
    }
    void avgpool(const float* in, int H, int W, int C, float* out) {
        begin(CLS_AVGPOOL);
        k_avgpool2<<<m->sms * 4, 256, 0, st>>>(in, H, W, C, d_n, off, cap, out);
        end();
    }
    // MobileNetV2: 3x3 stride-2 stem and the depthwise 3x3 of an inverted-residual block
    void stem3(const float* blob, const float* w, const float* bias, int C0, float* out) {
        begin(CLS_STEM);
        k_stem3<<<m->sms * 8, 256, 0, st>>>(blob, w, bias, C0, d_n, off, cap, out);
        end();
    }
    void dwconv3(const float* in, int H, int W, int C, int stride, const float* w9c, const float* bias, float* out) {
        begin(CLS_LIGHTCONV);
        k_dwconv3<<<m->sms * 8, 256, 0, st>>>(in, H, W, C, stride, w9c, bias, d_n, off, cap, out);
        end();
    }
    // LMBN_n head: the poolings of one branch output, the neck GEMMs of the chunk, the row L2 normalisation
    void lmbn_pool(const float* x, int H, int W, int which, float* pooled) {
        begin(CLS_HEAD);
        k_lmbn_pool<<<upper, 256, 0, st>>>(x, H, W, LMBN_C, which, pooled, d_n, off, cap);
        end();
    }
    void lmbn_neck(const NeckArgs& na, const float* pooled, const CropDesc* crops, float* out, int out_ld) {
        RCUDA_OK(cudaFuncSetAttribute(k_lmbn_neck, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)NECK_SMEM));
        begin(CLS_HEAD);
        k_lmbn_neck<<<dim3(LMBN_C / NECK_COLS, 6), 256, NECK_SMEM, st>>>(na, pooled, crops, d_n, off, cap, out, out_ld);
        end();
    }
    void l2_normalise(const CropDesc* crops, float* out, int out_ld, int feat) {
        begin(CLS_HEAD);
        k_l2_normalise<<<upper, 256, 0, st>>>(crops, d_n, off, cap, out, out_ld, feat);
        end();
    }
    void light(const LightArgs& a, int n_branches, int threads) {
        if (m->light_v2 && light2(a, n_branches)) return;
        inst[0] = 1; inst[1] = a.C; inst[2] = a.W; inst[3] = a.R;
        const int tiles = (a.H + a.R - 1) / a.R;
        const int n_grp = threads / (a.C / 4);
        const size_t smem = sizeof(float) * ((size_t)(a.R + 2) * (a.W + 2) * a.C + (size_t)a.C * a.C + 9 * a.C +
                                             (size_t)n_grp * a.C);
        if (smem > 48 * 1024)
            RCUDA_OK(cudaFuncSetAttribute(k_lightconv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        begin(CLS_LIGHTCONV);
        k_lightconv<<<dim3(tiles, n_branches, upper), threads, smem, st>>>(a, d_n, off, cap);
        end();
    }
};

// v2 keeps the staged input and the 1x1 result side by side: aim for two CTAs per SM, fall back to one
int pick_tile_rows2(int H, int W, int C) {
    for (size_t budget : {(size_t)100 * 1024, (size_t)220 * 1024})
        for (int R = H; R >= 1; --R) {
            if (H % R || R > 16) continue;
            if (light2_smem_bytes((R + 2) * (W + 2), C, 256) <= budget) return R;
        }
    return 1;
}

int pick_tile_rows(int H, int W, int C) {
    // largest divisor of H whose haloed tile (+ weights) stays under ~96 KB
    for (int R = H; R >= 1; --R) {
        if (H % R) continue;
        const size_t bytes = sizeof(float) * ((size_t)(R + 2) * (W + 2) * C + (size_t)C * C + 9 * C + 64 * C);
        if (bytes <= 96 * 1024 && R <= 16) return R;
    }
    return 1;
}

// Debug taps: stage index i stops the chunk after the i-th tapped tensor and leaves it in m->debug_ptr.
struct StageTaps {
    ReidModel* m;
    int idx = 0;
    bool operator()(const float* ptr, size_t per_crop) {
        if (m->debug_stop == idx++) { m->debug_ptr = ptr; m->debug_floats_per_crop = per_crop; return true; }
        return false;
    }
};

struct FrameIn {
    const uint8_t* images;
    size_t image_stride;
    int rows, cols;
    const CropDesc* crops;
};

// Crop staging of one chunk: every crop resized (or letterboxed) to in_h x in_w and normalised into m->blob
void stage_crops(Launcher& L, const FrameIn& fi) {
    ReidModel* m = L.m;
    L.begin(CLS_CROP);
    k_crop_resize_norm<<<L.upper, 256, 0, L.st>>>(fi.images, fi.image_stride, fi.rows, fi.cols, fi.crops, L.d_n, L.off,
                                                  L.cap, m->blob, m->preprocess, m->in_h, m->in_w, m->norm);
    L.end();
}

// Crop staging, 7x7 stem and 3x3 max pool of one chunk (taps 0-2): the pooled map (in_h/4 x 32 x c0) ends in m->bufB.
// Returns true when a debug tap stopped the chunk.
bool run_front(Launcher& L, const FrameIn& fi, StageTaps& stop_here) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    stage_crops(L, fi);
    if (stop_here(m->blob, (size_t)m->in_h * IN_W * 3)) return true;
    if (m->stem_in) {   // conv 7x7 -> IN -> ReLU -> max pool: the norm and the ReLU are applied inside the pool
        L.stem(true, m->blob, W + m->stem_w, nullptr, m->c[0], m->bufA, m->in_h);
        const int HW = (m->in_h / 2) * 64;
        double2* stats = reinterpret_cast<double2*>(m->sums[0]);
        L.in_stats(m->bufA, HW, m->c[0], stats, CLS_MAXPOOL);
        if (m->debug_stop == 1) {   // the stem tap is the map after IN + ReLU, which the fused pool never writes
            L.in_apply(m->bufA, nullptr, m->bufA, HW, m->c[0], W + m->stem_b, W + m->stem_beta, stats, 1, CLS_MAXPOOL);
            return stop_here(m->bufA, (size_t)HW * m->c[0]);   // tap 1
        }
        ++stop_here.idx;   // tap 1 is only materialised when it is the one asked for
        L.begin(CLS_MAXPOOL);
        k_maxpool3s2_in<<<m->sms * 8, 256, 0, L.st>>>(m->bufA, m->in_h / 2, 64, m->c[0], W + m->stem_b, W + m->stem_beta,
                                                      stats, L.d_n, L.off, L.cap, m->bufB);
        L.end();
        return stop_here(m->bufB, (size_t)(m->in_h / 4) * 32 * m->c[0]);
    }
    L.stem(false, m->blob, W + m->stem_w, W + m->stem_b, m->c[0], m->bufA, m->in_h);
    if (stop_here(m->bufA, (size_t)(m->in_h / 2) * 64 * m->c[0])) return true;
    L.maxpool(m->bufA, m->in_h / 2, 64, m->c[0], m->bufB);
    return stop_here(m->bufB, (size_t)(m->in_h / 4) * 32 * m->c[0]);
}

// One OSBlock (osnet.py:213-260): conv1 -> the four LightConv3x3 branches -> shared ChannelGate -> conv3 (+ downsample,
// or the identity) + ReLU.  X [crops][H][Wd][cin] -> Xo [crops][H][Wd][cout] (Xo != X); scratch m->x1, m->Y, m->sums,
// m->gates (and m->in_tmp).  b.in_mode places an instance norm before (OSNet-AIN) or after (OSNet-IBN) the residual
// add; IN_NONE launches exactly the OSNet sequence.
void run_osblock(Launcher& L, const BlockW& b, const float* X, float* Xo, int H, int Wd) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const int HW = H * Wd;
    PwArgs p{};
    p.in = X; p.w = W + b.c1w; p.bias = W + b.c1b; p.out = m->x1;
    p.K = b.cin; p.N = b.mid; p.HW = HW; p.relu = 1;
    p.w_tc = b.tc_c1.w; p.Kpad = b.tc_c1.Kpad; p.Npad = b.tc_c1.Npad;
    L.pointwise(p);
    int R = 0;
    if (m->light_chain && m->light_v2) {
        ChainArgs ca{};
        ca.in = m->x1; ca.H = H;
        for (int br = 0; br < 4; ++br) { ca.out[br] = m->Y[br][kDepth[br] & 1]; ca.sums[br] = m->sums[br]; }
        for (int l = 0; l < 10; ++l) {
            ca.wpw[l] = W + b.light[l].pw; ca.wdw[l] = W + b.light[l].dw; ca.bias[l] = W + b.light[l].b;
        }
        R = L.light_chain(ca, b.mid, Wd);
    }
    const bool chained = R > 0;
    if (!chained) R = m->light_v2 ? pick_tile_rows2(H, Wd, b.mid) : pick_tile_rows(H, Wd, b.mid);
    if (!chained && m->light_small && m->light_v2 && b.mid == 16 && Wd == 32) R = 8;
    const int tiles = H / R;
    const int threads = (256 / (b.mid / 4)) * (b.mid / 4);  // a multiple of the channel groups
    for (int level = 1; level <= 4 && !chained; ++level) {
        LightArgs la{};
        la.H = H; la.W = Wd; la.C = b.mid; la.R = R;
        int nb = 0;
        for (int l = 0; l < 10; ++l) {
            if (kLevelOfLight[l] != level) continue;
            const int br = kBranchOfLight[l];
            la.in[nb] = level == 1 ? m->x1 : m->Y[br][(level - 1) & 1];
            la.out[nb] = m->Y[br][level & 1];
            la.wpw[nb] = W + b.light[l].pw;
            la.wdw[nb] = W + b.light[l].dw;
            la.bias[nb] = W + b.light[l].b;
            la.wtc[nb] = b.light_tc[l].w;
            la.sums[nb] = kDepth[br] == level ? m->sums[br] : nullptr;
            ++nb;
        }
        L.light(la, nb, threads);
    }
    GateArgs ga{};
    for (int br = 0; br < 4; ++br) ga.sums[br] = m->sums[br];
    ga.w1 = W + b.g1w; ga.b1 = W + b.g1b; ga.w2 = W + b.g2w; ga.b2 = W + b.g2b;
    ga.gates = m->gates; ga.C = b.mid; ga.hid = b.hid; ga.tiles = tiles; ga.HW = HW;
    L.gates(ga);
    PwArgs c{};
    for (int br = 0; br < 4; ++br) c.branch[br] = m->Y[br][kDepth[br] & 1];
    c.gates = m->gates; c.mid = b.mid;
    if (b.in_mode == IN_BEFORE_RESIDUAL) {
        // OSBlockINin (osnet_ain.py): out = relu(IN(conv3(x2)) + identity').  conv3 (no bias, no ReLU) goes to a
        // cout-wide scratch (Xo itself when the identity is X); the downsample GEMM writes Xo; the norm pass reads both.
        float* x3 = b.has_ds ? m->in_tmp : Xo;
        c.w = W + b.cw; c.bias = W + b.cb; c.out = x3;
        c.K = b.mid; c.N = b.cout; c.HW = HW; c.relu = 0;
        L.pointwise(c);
        if (b.has_ds) {
            PwArgs d{};
            d.in = X; d.w = W + b.dsw; d.bias = W + b.dsb; d.out = Xo;
            d.K = b.cin; d.N = b.cout; d.HW = HW; d.relu = 0;
            L.pointwise(d);
        }
        double2* stats = reinterpret_cast<double2*>(m->sums[0]);
        L.in_stats(x3, HW, b.cout, stats, CLS_POINTWISE);
        L.in_apply(x3, b.has_ds ? Xo : X, Xo, HW, b.cout, W + b.ing, W + b.inb, stats, 1, CLS_POINTWISE);
        return;
    }
    c.in = b.has_ds ? X : nullptr;
    c.residual = b.has_ds ? nullptr : X;
    c.w = W + b.cw; c.bias = W + b.cb; c.out = Xo;
    c.K = b.mid + (b.has_ds ? b.cin : 0); c.N = b.cout; c.HW = HW; c.relu = 1;
    c.w_tc = b.tc_c.w; c.Kpad = b.tc_c.Kpad; c.Npad = b.tc_c.Npad;
    if (b.in_mode == IN_AFTER_RESIDUAL) c.relu = 0;   // OSBlock(IN=True): out = relu(IN(conv3(x2) + identity'))
    L.pointwise(c);
    if (b.in_mode == IN_AFTER_RESIDUAL) {
        double2* stats = reinterpret_cast<double2*>(m->sums[0]);
        L.in_stats(Xo, HW, b.cout, stats, CLS_POINTWISE);
        L.in_apply(Xo, nullptr, Xo, HW, b.cout, W + b.ing, W + b.inb, stats, 1, CLS_POINTWISE);
    }
}

// Transition (osnet.py conv2[2], conv3[2]): 1x1 + folded BN + ReLU of X [crops][H][Wd][C] into tmp, then 2x2 average
// pool into out [crops][H/2][Wd/2][C] (out may be X).
void run_transition(Launcher& L, const float* X, float* tmp, float* out, int H, int Wd, int C, size_t w, size_t bias,
                    const TcW& tc) {
    ReidModel* m = L.m;
    PwArgs p{};
    p.in = X; p.w = m->d_w + w; p.bias = m->d_w + bias; p.out = tmp;
    p.K = C; p.N = C; p.HW = H * Wd; p.relu = 1;
    p.w_tc = tc.w; p.Kpad = tc.Kpad; p.Npad = tc.Npad;
    L.pointwise(p);
    L.avgpool(tmp, H, Wd, C, out);
}

// LMBN_n, one chunk (lmbn_n.py:83-146 in eval).  Taps: 0 crop, 1 stem, 2 pool, 3 backone.2.0, 4 backone.2.1,
// 5 backone.2.2, 6 trunk end (backone.3), then per branch in the order global, bottleneck, partial, channel:
// 7-11 global .0.1, .0.2, .1.0, .1.1, .2 (branch end), 12 bottleneck, 13-17 partial, 18-22 channel.
void run_lmbn_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const LmbnW& lm = m->lm;
    StageTaps stop_here{m};
    if (run_front(L, fi, stop_here)) return;
    float* A = m->bufA;
    float* B = m->bufB;
    int H = m->in_h / 4, Wd = 32;
    run_osblock(L, lm.trunk[0], B, A, H, Wd);
    if (stop_here(A, (size_t)H * Wd * 256)) return;
    run_osblock(L, lm.trunk[1], A, B, H, Wd);
    if (stop_here(B, (size_t)H * Wd * 256)) return;
    run_transition(L, B, A, B, H, Wd, 256, lm.trunk_tw, lm.trunk_tb, TcW{});
    H /= 2; Wd /= 2;
    if (stop_here(B, (size_t)H * Wd * 256)) return;
    run_osblock(L, lm.trunk[2], B, m->trunk, H, Wd);
    if (stop_here(m->trunk, (size_t)H * Wd * 384)) return;
    const int bh = H / 2, bw = Wd / 2;   // branch maps after their transition: 24 x 8
    for (int br = 0; br < 3; ++br) {
        run_osblock(L, lm.br[br][0], m->trunk, A, H, Wd);
        if (stop_here(A, (size_t)H * Wd * 384)) return;
        run_transition(L, A, B, A, H, Wd, 384, lm.br_tw[br], lm.br_tb[br], TcW{});
        if (stop_here(A, (size_t)bh * bw * 384)) return;
        run_osblock(L, lm.br[br][1], A, B, bh, bw);
        if (stop_here(B, (size_t)bh * bw * LMBN_C)) return;
        run_osblock(L, lm.br[br][2], B, A, bh, bw);
        if (stop_here(A, (size_t)bh * bw * LMBN_C)) return;
        PwArgs p{};   // conv5
        p.in = A; p.w = m->d_w + lm.br_c5w[br]; p.bias = m->d_w + lm.br_c5b[br]; p.out = B;
        p.K = LMBN_C; p.N = LMBN_C; p.HW = bh * bw; p.relu = 1;
        L.pointwise(p);
        if (stop_here(B, (size_t)bh * bw * LMBN_C)) return;
        const float* pool_src = B;
        if (br == 0) {   // BatchFeatureErase_Top in eval: the bottleneck OSBlock; glo and glo_drop are its output
            run_osblock(L, lm.bottleneck, B, A, bh, bw);
            if (stop_here(A, (size_t)bh * bw * LMBN_C)) return;
            pool_src = A;
        }
        L.lmbn_pool(pool_src, bh, bw, br, m->pooled);
    }
    NeckArgs na{};
    for (int k = 0; k < 5; ++k) { na.w[k] = m->d_w + lm.neck_w[k]; na.b[k] = m->d_w + lm.neck_b[k]; }
    na.wsh = m->d_w + lm.sh_w; na.bsh = m->d_w + lm.sh_b; na.chst = m->d_w + lm.ch_st;
    L.lmbn_neck(na, m->pooled, fi.crops, d_out, out_ld);
    L.l2_normalise(fi.crops, d_out, out_ld, m->feat);
}

// Bottleneck ResNet, one chunk (resnet.py featuremaps + global average pool).  Taps: 0 crop, 1 stem, 2 pool, then
// 3 + i after Bottleneck i (layer1.0 first).  Per Bottleneck: conv1 (1x1) and conv2 (3x3, the block's stride) with
// bias + ReLU, then conv3 with the residual: block 0 of a stage runs conv3 and the strided downsample as one GEMM over
// [conv2 out | x], the others add x in the epilogue.  The head pools layer4 and L2-normalises into the caller's rows.
void run_resnet_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    StageTaps stop_here{m};
    if (run_front(L, fi, stop_here)) return;
    float* X = m->bufB;
    float* Xo = m->bufA;
    int H = IN_H / 4, Wd = IN_W / 4;
    for (const RnBlock& b : m->rn) {
        const int Ho = H / b.stride, Wo = Wd / b.stride;
        rn::ConvArgs c{};
        c.in0 = X; c.H0 = H; c.W0 = Wd; c.C0 = b.cin; c.k0 = 1; c.s0 = 1;
        c.w = b.c1.w; c.bias = W + b.c1.b; c.out = m->x1; c.Ho = H; c.Wo = Wd; c.N = b.width; c.relu = 1;
        L.conv_tc(c);
        c = rn::ConvArgs{};
        c.in0 = m->x1; c.H0 = H; c.W0 = Wd; c.C0 = b.width; c.k0 = 3; c.s0 = b.stride;
        c.w = b.c2.w; c.bias = W + b.c2.b; c.out = m->Y[0][0]; c.Ho = Ho; c.Wo = Wo; c.N = b.width; c.relu = 1;
        L.conv_tc(c);
        c = rn::ConvArgs{};
        c.in0 = m->Y[0][0]; c.H0 = Ho; c.W0 = Wo; c.C0 = b.width; c.k0 = 1; c.s0 = 1;
        if (b.cin != b.cout || b.stride != 1) {
            c.in1 = X; c.H1 = H; c.W1 = Wd; c.C1 = b.cin; c.s1 = b.stride;
        } else {
            c.residual = X;
        }
        c.w = b.c3.w; c.bias = W + b.c3.b; c.out = Xo; c.Ho = Ho; c.Wo = Wo; c.N = b.cout; c.relu = 1;
        L.conv_tc(c);
        std::swap(X, Xo);
        H = Ho; Wd = Wo;
        if (stop_here(X, (size_t)H * Wd * b.cout)) return;
    }
    L.head(X, H * Wd, m->feat, nullptr, nullptr, m->feat, fi.crops, d_out, out_ld);
}

// CLIP-ReID ViT-B/16, one chunk (clip/model.py VisionTransformer.forward + make_model.py build_transformer, eval,
// NECK_FEAT "after").  Taps: 0 crop, 1 patch embedding ([P][768]), 2 ln_pre ([T][768]), 3 + l after residual block l,
// 3 + layers the un-normalised 1280-d head row.  Every linear layer is rn::k_conv_tc over a [crops x T] x 1 map; the
// two residual adds run in the epilogues of out_proj and c_proj, in place on the stream (each element is read and
// written by the same thread).  Timing classes: crop, stem (patchify + patch GEMM), gates (LayerNorm), pointwise_gemm
// (linear layers), lightconv (attention), head.
void run_clip_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const VitW& v = m->vit;
    constexpr int D = vit::D;
    const int T = v.tokens, P = T - 1;
    StageTaps stop_here{m};
    stage_crops(L, fi);
    if (stop_here(m->blob, (size_t)m->in_h * m->in_w * 3)) return;
    float* X = m->bufA;          // residual stream [T][768]
    float* Xn = m->bufB;         // LayerNorm output
    float* att = m->Y[0][0];     // attention output / patch embedding
    float* hid = m->Y[0][1];     // MLP hidden layer / patch rows
    float* qkv = m->x1;
    L.begin(CLS_STEM);
    vit::k_vit_patchify<<<m->sms * 8, 256, 0, L.st>>>(m->blob, m->in_h, m->in_w, vit::PATCH, L.d_n, L.off, L.cap, hid);
    L.end();
    auto linear = [&](const float* in, int K, const float* w, const float* bias, const float* residual, int N, int act,
                      float* out, int rows) {
        rn::ConvArgs c{};
        c.in0 = in; c.H0 = rows; c.W0 = 1; c.C0 = K; c.k0 = 1; c.s0 = 1;
        c.w = w; c.bias = bias; c.residual = residual; c.out = out; c.Ho = rows; c.Wo = 1; c.N = N; c.relu = act;
        L.conv_tc(c);
    };
    linear(hid, 3 * vit::PATCH * vit::PATCH, v.patch_w, W + v.patch_b, nullptr, D, 0, att, P);
    if (stop_here(att, (size_t)P * D)) return;
    L.vit_layernorm(true, att, W + v.pos, W + v.lnpre_g, W + v.lnpre_b, T, X);
    if (stop_here(X, (size_t)T * D)) return;
    for (const VitLayer& l : v.layer) {
        L.vit_layernorm(false, X, nullptr, W + l.ln1g, W + l.ln1b, T, Xn);
        linear(Xn, D, l.win, W + l.bin, nullptr, 3 * D, 0, qkv, T);
        L.vit_attention(qkv, T, att);
        linear(att, D, l.wout, W + l.bout, X, D, 0, X, T);
        L.vit_layernorm(false, X, nullptr, W + l.ln2g, W + l.ln2b, T, Xn);
        linear(Xn, D, l.wfc, W + l.bfc, nullptr, 4 * D, 2, hid, T);
        linear(hid, 4 * D, l.wproj, W + l.bproj, X, D, 0, X, T);
        if (stop_here(X, (size_t)T * D)) return;
    }
    const bool tap = m->debug_stop == 3 + v.layers;
    L.begin(CLS_HEAD);
    vit::k_vit_head<<<L.upper, 256, 0, L.st>>>(X, T, W + v.head_g, W + v.head_b, W + v.head_w, W + v.head_pb, fi.crops,
                                               L.d_n, L.off, L.cap, d_out, out_ld, tap ? Xn : nullptr);
    L.end();
    if (tap) stop_here(Xn, vit::FEAT);
}

// ViT-Nano / ViT-Tiny, one chunk (vit_nano.py ViTNano.forward / vit_tiny.py ViTTinyParts.forward, eval).  Taps: 0 crop,
// 1 patch embedding ([P][192]), 2 tokens ([T][192]), 3 + l after block l, 3 + depth the final norm, 4 + depth the head
// row before the L2 norm.  Per block: norm1 (LayerNorm, or AdaptiveINLN in the first `ain` blocks), qkv, attention,
// proj + residual, norm2, fc1 + GELU, fc2 + residual; the linear layers are rn::k_conv_tc over a [crops x T] x 1 map
// with the residual adds in place in the epilogue, as for CLIP.  Timing classes: crop, stem (patchify, patch GEMM,
// tokens), gates (norms), pointwise_gemm (linear layers), lightconv (attention), head.
void run_vits_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const VitsW& v = m->vs;
    constexpr int D = vits::D;
    const int T = v.tokens, P = T - 1;
    StageTaps stop_here{m};
    stage_crops(L, fi);
    if (stop_here(m->blob, (size_t)m->in_h * m->in_w * 3)) return;
    float* X = m->bufA;          // residual stream [T][192]
    float* Xn = m->bufB;         // norm output
    float* att = m->Y[0][0];     // attention output / patch embedding
    float* hid = m->Y[0][1];     // MLP hidden layer / patch rows
    float* qkv = m->x1;
    L.begin(CLS_STEM);
    vit::k_vit_patchify<<<m->sms * 8, 256, 0, L.st>>>(m->blob, m->in_h, m->in_w, v.stride, L.d_n, L.off, L.cap, hid);
    L.end();
    auto linear = [&](const float* in, int K, const float* w, const float* bias, const float* residual, int N, int act,
                      float* out, int rows) {
        rn::ConvArgs c{};
        c.in0 = in; c.H0 = rows; c.W0 = 1; c.C0 = K; c.k0 = 1; c.s0 = 1;
        c.w = w; c.bias = bias; c.residual = residual; c.out = out; c.Ho = rows; c.Wo = 1; c.N = N; c.relu = act;
        L.conv_tc(c);
    };
    linear(hid, 3 * vit::PATCH * vit::PATCH, v.patch_w, W + v.patch_b, nullptr, D, 0, att, P);
    if (stop_here(att, (size_t)P * D)) return;
    L.begin(CLS_STEM);
    vits::k_vits_tokens<<<m->sms * 8, 256, 0, L.st>>>(att, W + v.pos, T, L.d_n, L.off, L.cap, X);
    L.end();
    if (stop_here(X, (size_t)T * D)) return;
    for (const VitsLayer& l : v.layer) {
        if (l.ain) L.vits_ain(X, W + l.n1a, W + l.n1b, W + l.n1c, T, Xn);
        else L.vits_layernorm(X, W + l.n1a, W + l.n1b, T, Xn);
        linear(Xn, D, l.wqkv, W + l.bqkv, nullptr, 3 * D, 0, qkv, T);
        L.vit_attention(qkv, T, att, D);
        linear(att, D, l.wproj, W + l.bproj, X, D, 0, X, T);
        L.vits_layernorm(X, W + l.n2g, W + l.n2b, T, Xn);
        linear(Xn, D, l.wfc1, W + l.bfc1, nullptr, vits::MLP, 4, hid, T);
        linear(hid, vits::MLP, l.wfc2, W + l.bfc2, X, D, 0, X, T);
        if (stop_here(X, (size_t)T * D)) return;
    }
    L.vits_layernorm(X, W + v.norm_g, W + v.norm_b, T, Xn);
    if (stop_here(Xn, (size_t)T * D)) return;
    const bool tap = m->debug_stop == stop_here.idx;
    L.vits_head(Xn, T, v.gh, v.gw, v.pool, v.proj, W + v.head, fi.crops, d_out, out_ld, tap ? qkv : nullptr);
    if (tap) stop_here(qkv, m->feat);
}

// MLFN, one chunk (mlfn.py MLFN.forward, eval).  Taps: 0 crop, 1 stem, 2 pool, 3 + i after MLFNBlock i, 19 s_hat
// ([512]), 20 the head row v = 0.5 (x + s) before the L2 norm ([1024]).  Per block: the FSM (average pool of x, two
// 1x1 layers + ReLU on k_conv_tc over a [crops] x 1 map, the last layer + sigmoid into s_hat), fm_conv1 (+ ReLU), the
// grouped 3x3 with the block's gates, the strided downsample (first block of a stage) into the output buffer, and
// fm_conv3 with the relu(residual + relu(.)) epilogue.  The head pools the last map, runs fc_x (+ ReLU), and fc_s with
// the same epilogue and fc_x's output as the residual (x >= 0, so the outer ReLU leaves x + s), then halves,
// L2-normalises and scatters.  Timing classes as for ResNet: 1x1 convolutions `pointwise_gemm`, the grouped 3x3
// `lightconv`, pools and gates `gates`, the head's last kernel `head`.
void run_mlfn_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const MlfnW& ml = m->ml;
    StageTaps stop_here{m};
    if (run_front(L, fi, stop_here)) return;
    auto conv1x1 = [&](const float* in, int h, int w, int cin, int stride, const RnConv& cv, int N, const float* res,
                       int act, float* out) {
        rn::ConvArgs c{};
        c.in0 = in; c.H0 = h; c.W0 = w; c.C0 = cin; c.k0 = 1; c.s0 = stride;
        c.w = cv.w; c.bias = W + cv.b; c.residual = res; c.out = out;
        c.Ho = (h - 1) / stride + 1; c.Wo = (w - 1) / stride + 1; c.N = N; c.relu = act;
        L.conv_tc(c);
    };
    float* X = m->bufB;
    float* Xo = m->bufA;
    int H = IN_H / 4, Wd = IN_W / 4, col = 0;
    for (const MlfnBlock& b : ml.blocks) {
        L.mlfn_gap(X, H * Wd, b.cin, m->pooled);
        conv1x1(m->pooled, 1, 1, b.cin, 1, b.fsm1, b.f0, nullptr, 1, m->sums[0]);
        conv1x1(m->sums[0], 1, 1, b.f0, 1, b.fsm2, b.f1, nullptr, 1, m->sums[1]);
        L.mlfn_gate(m->sums[1], b.f1, W + b.fsm3w, W + b.fsm3b, m->gates, col);
        conv1x1(X, H, Wd, b.cin, 1, b.c1, b.mid, nullptr, 1, m->x1);
        L.group_conv(m->x1, H, Wd, b.mid, b.gw, b.stride, W + b.gcw, W + b.gcb, m->gates + col, m->Y[0][0]);
        const int Ho = H / b.stride, Wo = Wd / b.stride;
        if (b.ds) conv1x1(X, H, Wd, b.cin, b.stride, b.down, b.cout, nullptr, 0, Xo);
        conv1x1(m->Y[0][0], Ho, Wo, b.mid, 1, b.c3, b.cout, b.ds ? Xo : X, 3, Xo);
        std::swap(X, Xo);
        H = Ho; Wd = Wo; col += mlfn::GROUPS;
        if (stop_here(X, (size_t)H * Wd * b.cout)) return;
    }
    if (stop_here(m->gates, mlfn::SHAT)) return;
    L.mlfn_gap(X, H * Wd, 2048, m->pooled);
    conv1x1(m->pooled, 1, 1, 2048, 1, ml.fc_x, mlfn::FEAT, nullptr, 1, m->sums[2]);
    conv1x1(m->gates, 1, 1, mlfn::SHAT, 1, ml.fc_s, mlfn::FEAT, m->sums[2], 3, m->sums[3]);
    const bool tap = m->debug_stop == stop_here.idx;
    L.begin(CLS_HEAD);
    mlfn::k_mlfn_head<<<L.upper, 256, 0, L.st>>>(m->sums[3], fi.crops, L.d_n, L.off, L.cap, d_out, out_ld,
                                                 tap ? m->sums[2] : nullptr);
    L.end();
    if (tap) stop_here(m->sums[2], mlfn::FEAT);
}

hacnn::AttnW hacnn_attn_w(const float* W, const size_t* o) {
    return hacnn::AttnW{W + o[0], W + o[1], W + o[2], W + o[3], W + o[4], W + o[5], W + o[6], W + o[7], W + o[8]};
}

// HACNN, one chunk (hacnn.py HACNN.forward, eval).  Taps: 0 crop (160x64x3), 1 stem (80x32x32), 2 + i x_{i+1}_out
// (i = 0 .. 2: 40x16x128, 20x8x256, 10x4x384), 5 + i the local map of level i + 1 ([region][h][w][C]: 4 x 12x14x128,
// 4 x 6x7x256, 4 x 3x4x384), 8 theta ([level][region][tx, ty], 24), 9 the head row [fc_global | fc_local] before the
// normalisations (1024).  Per level: InceptionA and InceptionB on k_conv_tc, every stream storing its slice of the
// concatenated map; the attention (s, v, theta) of the InceptionB output; the STN of the previous level's output
// (the stem for level 1) resized and added to the previous local map; the local InceptionB over the chunk's
// 4 x crops regions (a second Launcher whose device count is 4 x the crop count); then x *= attention.  The head
// pools both branches, runs fc_global / fc_local (BatchNorm1d folded, ReLU) on k_conv_tc over a [crops] x 1 map into
// the two halves of the head row, and normalises.  Timing classes: 1x1 `pointwise_gemm`, 3x3 `lightconv`, pools
// `maxpool` / `avgpool`, attention and STN `gates`, the head `head`.
void run_hacnn_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const HacnnW& h = m->ha;
    auto tap = [&](int idx, const float* p, size_t per_crop) {
        if (m->debug_stop != idx) return false;
        m->debug_ptr = p;
        m->debug_floats_per_crop = per_crop;
        return true;
    };
    stage_crops(L, fi);
    if (tap(0, m->blob, (size_t)hacnn::IN_H * hacnn::IN_W * 3)) return;
    L.hacnn_stem(m->blob, W + m->stem_w, W + m->stem_b, m->bufA);
    if (tap(1, m->bufA, (size_t)80 * 32 * hacnn::STEM_C)) return;
    L.begin(CLS_GATES);
    hacnn::k_count4<<<1, 1, 0, L.st>>>(L.d_n, m->d_n4);
    L.end();
    Launcher R{m, m->d_n4, 4 * L.off, 4 * L.cap, 4 * L.upper, L.st};   // the local branch: [crop][region] images
    auto conv = [&](Launcher& La, const float* in, int H, int Wd, int cin, int k, int stride, const RnConv& cv, int N,
                    float* out, int ld) {
        rn::ConvArgs c{};
        c.in0 = in; c.H0 = H; c.W0 = Wd; c.C0 = cin; c.k0 = k; c.s0 = stride;
        c.w = cv.w; c.bias = W + cv.b; c.out = out;
        c.Ho = (H - 1) / stride + 1; c.Wo = (Wd - 1) / stride + 1; c.N = N; c.relu = 1; c.out_ld = ld;
        La.conv_tc(c);
    };
    auto inception_b = [&](Launcher& La, const RnConv* cv, const float* x, int H, int Wd, int cin, int cout, float* out) {
        const int mid = cout / 4;
        conv(La, x, H, Wd, cin, 1, 1, cv[0], mid, m->Y[0][0], mid);
        conv(La, m->Y[0][0], H, Wd, mid, 3, 2, cv[1], mid, out, cout);
        conv(La, x, H, Wd, cin, 1, 1, cv[2], mid, m->Y[0][0], mid);
        conv(La, m->Y[0][0], H, Wd, mid, 3, 1, cv[3], mid, m->Y[0][1], mid);
        conv(La, m->Y[0][1], H, Wd, mid, 3, 2, cv[4], mid, out + mid, cout);
        La.hacnn_pool(true, x, H, Wd, cin, m->Y[1][0]);
        conv(La, m->Y[1][0], (H - 1) / 2 + 1, (Wd - 1) / 2 + 1, cin, 1, 1, cv[5], 2 * mid, out + 2 * mid, cout);
    };
    static const int kC[4] = {hacnn::STEM_C, 128, 256, hacnn::C3};
    static const int kLocal[3][2] = {{24, 28}, {12, 14}, {6, 7}};
    float *prev = m->bufA, *cur = m->bufB, *T = m->Y[1][1], *Lc = m->Y[2][0];
    int H = 80, Wd = 32;
    for (int i = 0; i < 3; ++i) {
        const int cin = kC[i], c = kC[i + 1], mid = c / 4, Hc = H / 2, Wc = Wd / 2;
        for (int s = 0; s < 3; ++s) {   // InceptionA into x1, then InceptionB into cur
            conv(L, prev, H, Wd, cin, 1, 1, h.ia[i][2 * s], mid, m->Y[0][0], mid);
            conv(L, m->Y[0][0], H, Wd, mid, 3, 1, h.ia[i][2 * s + 1], mid, m->x1 + s * mid, c);
        }
        L.hacnn_pool(false, prev, H, Wd, cin, m->Y[1][0]);
        conv(L, m->Y[1][0], H, Wd, cin, 1, 1, h.ia[i][6], mid, m->x1 + 3 * mid, c);
        inception_b(L, h.ib[i], m->x1, H, Wd, c, c, cur);
        L.hacnn_attn(cur, Hc, Wc, c, hacnn_attn_w(W, h.att[i]), i, m->sums[0], m->sums[1], m->gates);
        const int lh = kLocal[i][0], lw = kLocal[i][1];
        L.hacnn_stn(prev, H, Wd, cin, m->gates + 8 * i, i ? Lc : nullptr, lh, lw, T);
        inception_b(R, h.lb[i], T, lh, lw, cin, c, Lc);
        L.hacnn_attn_apply(cur, Hc * Wc, c, m->sums[0], m->sums[1], W + h.att[i][6]);
        L.launches += R.launches;
        R.launches = 0;
        if (tap(2 + i, cur, (size_t)Hc * Wc * c) ||
            tap(5 + i, Lc, (size_t)4 * ((lh - 1) / 2 + 1) * ((lw - 1) / 2 + 1) * c))
            return;
        std::swap(prev, cur);
        H = Hc; Wd = Wc;
    }
    if (tap(8, m->gates, hacnn::THETA)) return;
    float* pg = m->pooled;
    float* pl = m->pooled + (size_t)m->chunk * hacnn::C3;
    L.hacnn_head_pool(prev, H * Wd, Lc, 3 * 4, pg, pl);
    conv(L, pg, 1, 1, hacnn::C3, 1, 1, h.fcg, hacnn::HALF, m->sums[2], hacnn::FEAT);
    conv(L, pl, 1, 1, 4 * hacnn::C3, 1, 1, h.fcl, hacnn::HALF, m->sums[2] + hacnn::HALF, hacnn::FEAT);
    if (tap(9, m->sums[2], hacnn::FEAT)) return;
    L.hacnn_head(m->sums[2], fi.crops, d_out, out_ld);
}

// CSPReID-n, one chunk (cspreid_n.py CSPReID_n.forward, eval).  Taps: 0 crop (H x W x 3), 1 stem (H/4 x W/4 x 64),
// 2-4 stages 1-3 after their downsample (H/8 x W/8 x 128, H/16 x W/16 x 256, H/32 x W/32 x 384), 5 stage 4's C3k2,
// 6 SPPF, 7 the attention (H/32 x W/32 x 512 each), 8 the interleaved head row before the L2 norm (1536).  Every
// ConvBNSiLU after the first stem conv runs on k_conv_tc's SILU instances.  A C3k2's cv1 stores both halves into the
// first 2 mid channels of its concatenation in m->x1; each bottleneck reads the previous slice in place (the chunk
// is free), writes its hidden map to Y[0][0] and its output, residual + SiLU(.), into the next slice (the cat is free);
// cv2 reads the whole concatenation.  SPPF's cv1 writes slice 0 of a 1024-wide concatenation and one launch fills
// slices 1-3 with the chained pools.  Timing classes: 1x1 `pointwise_gemm`, 3x3 `lightconv`, SPPF `maxpool`, the
// attention `gates`, the head `head`.
void run_cspreid_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const CspW& cs = m->cs;
    StageTaps stop_here{m};
    stage_crops(L, fi);
    if (stop_here(m->blob, (size_t)m->in_h * m->in_w * 3)) return;
    int i = 0;   // the next packed conv
    auto conv = [&](const float* in, int H, int Wd, int cin, int in_ld, int k, int stride, int N, const float* res,
                    int res_ld, float* out, int ld) {
        const RnConv& cv = cs.conv[i++];
        rn::ConvArgs c{};
        c.in0 = in; c.H0 = H; c.W0 = Wd; c.C0 = cin; c.k0 = k; c.s0 = stride; c.in_ld = in_ld;
        c.w = cv.w; c.bias = W + cv.b; c.residual = res; c.res_ld = res_ld; c.out = out; c.out_ld = ld;
        c.Ho = (H - 1) / stride + 1; c.Wo = (Wd - 1) / stride + 1; c.N = N; c.relu = res ? 6 : 5;
        L.conv_tc_silu(c);
    };
    L.csp_stem(m->blob, m->in_h, m->in_w, W + m->stem_w, W + m->stem_b, m->bufA);
    int H = m->in_h / 2, Wd = m->in_w / 2;
    conv(m->bufA, H, Wd, csp::STEM_C, csp::STEM_C, 3, 2, 64, nullptr, 0, m->bufB, 64);
    H = (H - 1) / 2 + 1; Wd = (Wd - 1) / 2 + 1;
    if (stop_here(m->bufB, (size_t)H * Wd * 64)) return;
    float* X = m->bufB;
    for (int s = 0; s < 4; ++s) {
        const int cin = kCspStage[s][0], cout = kCspStage[s][1], n = kCspStage[s][2], mid = cout / 2;
        const int ld = (2 + n) * mid;
        float* cat = m->x1;
        conv(X, H, Wd, cin, cin, 1, 1, 2 * mid, nullptr, 0, cat, ld);
        for (int b = 0; b < n; ++b) {
            float* src = cat + (1 + b) * mid;
            conv(src, H, Wd, mid, ld, 1, 1, mid / 2, nullptr, 0, m->Y[0][0], mid / 2);
            conv(m->Y[0][0], H, Wd, mid / 2, mid / 2, 3, 1, mid, src, ld, src + mid, ld);
        }
        conv(cat, H, Wd, ld, ld, 1, 1, cout, nullptr, 0, m->bufA, cout);
        if (s == 3) break;
        conv(m->bufA, H, Wd, cout, cout, 3, 2, cout, nullptr, 0, m->bufB, cout);
        H = (H - 1) / 2 + 1; Wd = (Wd - 1) / 2 + 1;
        if (stop_here(m->bufB, (size_t)H * Wd * cout)) return;
    }
    const size_t map = (size_t)H * Wd * csp::C;
    if (stop_here(m->bufA, map)) return;
    conv(m->bufA, H, Wd, csp::C, csp::C, 1, 1, csp::SPPF_C, nullptr, 0, m->x1, 4 * csp::SPPF_C);
    L.csp_sppf(m->x1, H, Wd, csp::SPPF_C);
    conv(m->x1, H, Wd, 4 * csp::SPPF_C, 4 * csp::SPPF_C, 1, 1, csp::C, nullptr, 0, m->bufB, csp::C);
    if (stop_here(m->bufB, map)) return;
    const float* attn[5] = {W + cs.attn[0], W + cs.attn[1], W + cs.attn[2], W + cs.attn[3], W + cs.attn[4]};
    L.csp_attn(m->bufB, H, Wd, attn, m->bufA);
    if (stop_here(m->bufA, map)) return;
    const float* head[6] = {W + cs.head[0], W + cs.head[1], W + cs.head[2], W + cs.head[3], W + cs.head[4],
                            W + cs.head[5]};
    const bool tap = m->debug_stop == stop_here.idx;
    L.csp_head(m->bufA, H, Wd, head, fi.crops, d_out, out_ld, tap ? m->sums[0] : nullptr);
    if (tap) stop_here(m->sums[0], csp::FEAT);
}

// MobileNetV2, one chunk: stem -> [expand 1x1 + ReLU6 -> depthwise 3x3 + ReLU6 -> project 1x1 (+ residual)] x 17 ->
// conv9 -> GAP.  No debug taps.
void run_mobilenetv2_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    const float* W = m->d_w;
    const MbW& mb = m->mb;
    stage_crops(L, fi);
    float* X = m->bufA;
    float* Xo = m->bufB;
    L.stem3(m->blob, W + mb.stem_w, W + mb.stem_b, mb.stemp, X);
    int H = 128, Wd = 64;
    for (const MbBlock& b : mb.blocks) {
        PwArgs e{};
        e.in = X; e.w = W + b.we; e.bias = W + b.be; e.out = m->x1;
        e.K = b.cinp; e.N = b.midp; e.HW = H * Wd; e.relu = 2;
        L.pointwise(e);
        L.dwconv3(m->x1, H, Wd, b.midp, b.stride, W + b.wd, W + b.bd, m->Y[0][0]);
        H /= b.stride; Wd /= b.stride;
        PwArgs p{};
        p.in = m->Y[0][0]; p.w = W + b.wp; p.bias = W + b.bp; p.out = Xo;
        p.residual = (b.stride == 1 && b.cin == b.cout) ? X : nullptr;
        p.K = b.midp; p.N = b.coutp; p.HW = H * Wd; p.relu = 0;
        L.pointwise(p);
        std::swap(X, Xo);
    }
    PwArgs c9{};
    c9.in = X; c9.w = W + mb.c9w; c9.bias = W + mb.c9b; c9.out = Xo;
    c9.K = mb.last; c9.N = m->feat; c9.HW = H * Wd; c9.relu = 2;
    L.pointwise(c9);
    L.head(Xo, H * Wd, m->feat, nullptr, nullptr, m->feat, fi.crops, d_out, out_ld);
}
}  // namespace

}  // namespace bmb
#include "reid_tc_plan.cuh"
namespace bmb {

namespace {
// OSNet head: global average pool of x [crops][HW][c3], fc + folded BatchNorm1d, L2 norm into the caller's rows
void run_osnet_head(Launcher& L, const FrameIn& fi, const float* x, int HW, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    L.head(x, HW, m->c[3], m->d_w + m->fcw, m->d_w + m->fcb, m->feat, fi.crops, d_out, out_ld);
}

// OSNet and OSNet-AIN / IBN, one chunk (osnet.py:380-405).  Taps: 0 crop, 1 stem, 2 pool, then every OSBlock and
// transition output in order, conv5 last.
void run_osnet_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    ReidModel* m = L.m;
    if (m->tc && m->debug_stop != 0 && m->debug_stop != 1) {
        // tensor-core path: crop staging, stem and max pool are one fused kernel (k_front_tc); diagnostic stops at the
        // blob / stem tensors (0, 1) run the float32 kernels below instead
        const tcx::FrontInput tfi{fi.images, fi.image_stride, fi.rows, fi.cols, fi.crops, d_out, out_ld};
        if (tcx::plan_run(m, tfi, L.d_n, L.off, L.upper, L.st, L)) return;
        if (!(m->tc->head_fused && m->debug_stop < 0)) run_osnet_head(L, fi, m->tc->c5, 128, d_out, out_ld);
        return;
    }
    StageTaps stop_here{m};
    if (run_front(L, fi, stop_here)) return;
    float* X = m->bufB;
    float* Xo = m->bufA;
    int H = 64, Wd = 32;
    for (int s = 0; s < 3; ++s) {
        for (int j = 0; j < 2; ++j) {
            const BlockW& b = m->blocks[s * 2 + j];
            run_osblock(L, b, X, Xo, H, Wd);
            std::swap(X, Xo);
            if (stop_here(X, (size_t)H * Wd * b.cout)) return;
        }
        if (s < 2) {
            const int C = m->c[s + 1];
            run_transition(L, X, Xo, X, H, Wd, C, m->trans_w[s], m->trans_b[s], m->tc_trans[s]);
            H /= 2; Wd /= 2;
            if (stop_here(X, (size_t)H * Wd * C)) return;
        }
    }
    const int C = m->c[3];
    PwArgs p{};
    p.in = X; p.w = m->d_w + m->c5w; p.bias = m->d_w + m->c5b; p.out = Xo;
    p.K = C; p.N = C; p.HW = H * Wd; p.relu = 1;
    p.w_tc = m->tc_c5.w; p.Kpad = m->tc_c5.Kpad; p.Npad = m->tc_c5.Npad;
    L.pointwise(p);
    if (stop_here(Xo, (size_t)H * Wd * C)) return;
    run_osnet_head(L, fi, Xo, H * Wd, d_out, out_ld);
}

void run_chunk(Launcher& L, const FrameIn& fi, float* d_out, int out_ld) {
    switch (L.m->arch) {
        case ARCH_OSNET:
        case ARCH_OSNET_IN: run_osnet_chunk(L, fi, d_out, out_ld); return;
        case ARCH_MOBILENETV2: run_mobilenetv2_chunk(L, fi, d_out, out_ld); return;
        case ARCH_LMBN_N: run_lmbn_chunk(L, fi, d_out, out_ld); return;
        case ARCH_RESNET: run_resnet_chunk(L, fi, d_out, out_ld); return;
        case ARCH_CLIP: run_clip_chunk(L, fi, d_out, out_ld); return;
        case ARCH_MLFN: run_mlfn_chunk(L, fi, d_out, out_ld); return;
        case ARCH_HACNN: run_hacnn_chunk(L, fi, d_out, out_ld); return;
        case ARCH_VIT: run_vits_chunk(L, fi, d_out, out_ld); return;
        case ARCH_CSPREID: run_cspreid_chunk(L, fi, d_out, out_ld); return;
    }
}
}  // namespace

int reid_forward(ReidModel* m, const uint8_t* d_images, size_t image_stride, int rows, int cols,
                 const CropDesc* d_crops, const int* d_ncrops, int max_crops, float* d_out, int out_ld,
                 cudaStream_t st, int first_crop, int last_crop) {
    // [first_crop, last_crop) restricts the call to a slice of the crop list (two models on two streams split a frame)
    if (last_crop < 0 || last_crop > max_crops) last_crop = max_crops;
    m->debug_ptr = nullptr;
    const FrameIn fi{d_images, image_stride, rows, cols, d_crops};
    int launches = 0;
    for (int off = first_crop; off < last_crop; off += m->chunk) {
        const int upper = (last_crop - off) < m->chunk ? (last_crop - off) : m->chunk;
        Launcher L{m, d_ncrops, off, upper, upper, st};
        run_chunk(L, fi, d_out, out_ld);
        launches += L.launches;
    }
    RCUDA_OK(cudaGetLastError());
    return launches;
}


// Standalone 1x1-convolution GEMM on host arrays (parity tests / micro-benchmarks): out = act(A W + bias (+ res)).
void standalone_pointwise(const float* A, int M, int K, const float* W, int N, const float* bias, const float* residual,
                          int relu, int use_tc, float* out, float* elapsed_ms) {
    if (M <= 0 || K <= 0 || N <= 0 || K % 4 || N % 4) throw std::runtime_error("M,K,N > 0 and K,N multiples of 4 required");
    float *dA = nullptr, *dW = nullptr, *dB = nullptr, *dR = nullptr, *dO = nullptr, *dWtc = nullptr;
    int* dn = nullptr;
    auto cleanup = [&] { cudaFree(dA); cudaFree(dW); cudaFree(dB); cudaFree(dR); cudaFree(dO); cudaFree(dWtc); cudaFree(dn); };
    try {
        RCUDA_OK(cudaMalloc(&dA, sizeof(float) * (size_t)M * K));
        RCUDA_OK(cudaMalloc(&dW, sizeof(float) * (size_t)K * N));
        RCUDA_OK(cudaMalloc(&dB, sizeof(float) * N));
        RCUDA_OK(cudaMalloc(&dO, sizeof(float) * (size_t)M * N));
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dA, A, sizeof(float) * (size_t)M * K, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dW, W, sizeof(float) * (size_t)K * N, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dB, bias, sizeof(float) * N, cudaMemcpyHostToDevice));
        if (residual) {
            RCUDA_OK(cudaMalloc(&dR, sizeof(float) * (size_t)M * N));
            RCUDA_OK(cudaMemcpy(dR, residual, sizeof(float) * (size_t)M * N, cudaMemcpyHostToDevice));
        }
        const int one = 1;
        RCUDA_OK(cudaMemcpy(dn, &one, sizeof(int), cudaMemcpyHostToDevice));
        ReidModel fake;
        fake.use_tc = use_tc != 0;
        PwArgs p{};
        p.in = dA; p.w = dW; p.bias = dB; p.residual = dR; p.out = dO; p.K = K; p.N = N; p.HW = M; p.relu = relu;
        if (use_tc) {
            if (M % tc::TILE_M) throw std::runtime_error("tensor-core path needs M % 128 == 0");
            const int Kpad = (K + 7) / 8 * 8, Npad = (N + 15) / 16 * 16;
            if (Npad > tc::NPAD_MAX || tc::smem_bytes(Kpad, Npad) > 200 * 1024) throw std::runtime_error("shape exceeds the tensor-core kernel's accumulators or shared memory");
            std::vector<float> packed(2 * (size_t)Npad * Kpad);
            tc::pack_weights(W, K, N, Kpad, Npad, packed.data());
            RCUDA_OK(cudaMalloc(&dWtc, sizeof(float) * packed.size()));
            RCUDA_OK(cudaMemcpy(dWtc, packed.data(), sizeof(float) * packed.size(), cudaMemcpyHostToDevice));
            p.w_tc = dWtc; p.Kpad = Kpad; p.Npad = Npad;
        }
        cudaEvent_t e0, e1;
        RCUDA_OK(cudaEventCreate(&e0));
        RCUDA_OK(cudaEventCreate(&e1));
        Launcher L{&fake, dn, 0, 1, 1, nullptr};
        L.pointwise(p);  // warm-up
        RCUDA_OK(cudaDeviceSynchronize());
        RCUDA_OK(cudaEventRecord(e0));
        for (int r = 0; r < 10; ++r) L.pointwise(p);
        RCUDA_OK(cudaEventRecord(e1));
        RCUDA_OK(cudaDeviceSynchronize());
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        if (elapsed_ms) *elapsed_ms = ms / 10.f;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * (size_t)M * N, cudaMemcpyDeviceToHost));
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

// Standalone instance norm on host arrays (parity tests): x [n][H][W][C] float32.
//   pool == 0: out [n][H][W][C] = act(IN(x) * gamma + beta (+ residual))     (k_in_stats + k_in_apply)
//   pool == 1: out [n][H/2][W/2][C] = maxpool3x3s2(relu(IN(x) * gamma + beta)) (k_in_stats + k_maxpool3s2_in)
void standalone_instance_norm(const float* x, int n, int H, int W, int C, const float* gamma, const float* beta,
                              const float* residual, int relu, int pool, float* out) {
    if (n <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 4 || (pool && (H % 2 || W % 2)))
        throw std::runtime_error("n, H, W, C > 0, C a multiple of 4 (and H, W even to pool) required");
    const size_t elems = (size_t)n * H * W * C, out_elems = pool ? elems / 4 : elems;
    float *dx = nullptr, *dg = nullptr, *db = nullptr, *dr = nullptr, *dout = nullptr;
    double2* dst = nullptr;
    int* dn = nullptr;
    auto cleanup = [&] { cudaFree(dx); cudaFree(dg); cudaFree(db); cudaFree(dr); cudaFree(dout); cudaFree(dst); cudaFree(dn); };
    try {
        RCUDA_OK(cudaMalloc(&dx, sizeof(float) * elems));
        RCUDA_OK(cudaMalloc(&dg, sizeof(float) * C));
        RCUDA_OK(cudaMalloc(&db, sizeof(float) * C));
        RCUDA_OK(cudaMalloc(&dout, sizeof(float) * out_elems));
        RCUDA_OK(cudaMalloc(&dst, sizeof(double2) * (size_t)n * C));
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dx, x, sizeof(float) * elems, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dg, gamma, sizeof(float) * C, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(db, beta, sizeof(float) * C, cudaMemcpyHostToDevice));
        if (residual && !pool) {
            RCUDA_OK(cudaMalloc(&dr, sizeof(float) * elems));
            RCUDA_OK(cudaMemcpy(dr, residual, sizeof(float) * elems, cudaMemcpyHostToDevice));
        }
        RCUDA_OK(cudaMemcpy(dn, &n, sizeof(int), cudaMemcpyHostToDevice));
        ReidModel fake;
        Launcher L{&fake, dn, 0, n, n, nullptr};
        L.in_stats(dx, H * W, C, dst, CLS_POINTWISE);
        if (pool)
            k_maxpool3s2_in<<<fake.sms * 8, 256>>>(dx, H, W, C, dg, db, dst, dn, 0, n, dout);
        else
            L.in_apply(dx, dr, dout, H * W, C, dg, db, dst, relu, CLS_POINTWISE);
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaDeviceSynchronize());
        RCUDA_OK(cudaMemcpy(out, dout, sizeof(float) * out_elems, cudaMemcpyDeviceToHost));
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

// Standalone ResNet convolution (rn::k_conv_tc) on host arrays (parity tests / micro-benchmarks):
//   out [n][Ho][Wo][N] = act(conv_k(in0, stride) (+ conv_1x1(in1, stride1)) + bias (+ residual)),
// in0 [n][h0][w0][c0] with k in {1, 3} (pad k / 2), in1 [n][h1][w1][c1] (c1 = 0: none), w [k*k*c0 + c1][N] K-major.
void standalone_resnet_conv(const float* in0, int n, int h0, int w0, int c0, int k, int stride, const float* in1, int h1,
                            int w1, int c1, int stride1, const float* w, int N, const float* bias, const float* residual,
                            int relu, float* out, float* elapsed_ms) {
    if (n <= 0 || h0 <= 0 || w0 <= 0 || c0 <= 0 || c0 % rn::KC || (k != 1 && k != 3) || stride < 1 || N <= 0 || N % 64 ||
        c1 < 0 || c1 % rn::KC || (c1 && (!in1 || h1 <= 0 || w1 <= 0 || stride1 < 1)) || relu < 0 || relu > 4 ||
        (relu == 3 && !residual))
        throw std::runtime_error("n, h0, w0 > 0, k in {1, 3}, c0 and c1 multiples of 32, N a multiple of 64, relu in "
                                 "{0, 1, 2, 3, 4} (3 with a residual) required");
    const int pad = k / 2, Ho = (h0 + 2 * pad - k) / stride + 1, Wo = (w0 + 2 * pad - k) / stride + 1;
    if (c1 && ((Ho - 1) * stride1 >= h1 || (Wo - 1) * stride1 >= w1))
        throw std::runtime_error("the second operand does not cover the output grid");
    const int K = k * k * c0 + c1;
    const size_t n_in0 = (size_t)n * h0 * w0 * c0, n_in1 = (size_t)n * h1 * w1 * c1, n_out = (size_t)n * Ho * Wo * N;
    float *d0 = nullptr, *d1 = nullptr, *dW = nullptr, *dB = nullptr, *dR = nullptr, *dO = nullptr;
    int* dn = nullptr;
    auto cleanup = [&] { cudaFree(d0); cudaFree(d1); cudaFree(dW); cudaFree(dB); cudaFree(dR); cudaFree(dO); cudaFree(dn); };
    try {
        std::vector<float> packed(2 * (size_t)K * N);
        rn::pack_conv_weights(w, K, N, packed.data());
        RCUDA_OK(cudaMalloc(&d0, sizeof(float) * n_in0));
        RCUDA_OK(cudaMemcpy(d0, in0, sizeof(float) * n_in0, cudaMemcpyHostToDevice));
        if (c1) {
            RCUDA_OK(cudaMalloc(&d1, sizeof(float) * n_in1));
            RCUDA_OK(cudaMemcpy(d1, in1, sizeof(float) * n_in1, cudaMemcpyHostToDevice));
        }
        RCUDA_OK(cudaMalloc(&dW, sizeof(float) * packed.size()));
        RCUDA_OK(cudaMemcpy(dW, packed.data(), sizeof(float) * packed.size(), cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMalloc(&dB, sizeof(float) * N));
        RCUDA_OK(cudaMemcpy(dB, bias, sizeof(float) * N, cudaMemcpyHostToDevice));
        if (residual) {
            RCUDA_OK(cudaMalloc(&dR, sizeof(float) * n_out));
            RCUDA_OK(cudaMemcpy(dR, residual, sizeof(float) * n_out, cudaMemcpyHostToDevice));
        }
        RCUDA_OK(cudaMalloc(&dO, sizeof(float) * n_out));
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dn, &n, sizeof(int), cudaMemcpyHostToDevice));
        rn::ConvArgs c{};
        c.in0 = d0; c.H0 = h0; c.W0 = w0; c.C0 = c0; c.k0 = k; c.s0 = stride;
        c.in1 = d1; c.H1 = h1; c.W1 = w1; c.C1 = c1; c.s1 = stride1;
        c.w = dW; c.bias = dB; c.residual = dR; c.out = dO; c.Ho = Ho; c.Wo = Wo; c.N = N; c.relu = relu;
        ReidModel fake;
        Launcher L{&fake, dn, 0, n, n, nullptr};
        L.conv_tc(c);   // warm-up
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaDeviceSynchronize());
        cudaEvent_t e0, e1;
        RCUDA_OK(cudaEventCreate(&e0));
        RCUDA_OK(cudaEventCreate(&e1));
        RCUDA_OK(cudaEventRecord(e0));
        for (int r = 0; r < 10; ++r) L.conv_tc(c);
        RCUDA_OK(cudaEventRecord(e1));
        RCUDA_OK(cudaDeviceSynchronize());
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        if (elapsed_ms) *elapsed_ms = ms / 10.f;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * n_out, cudaMemcpyDeviceToHost));
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

// Standalone CLIP LayerNorm (vit::k_vit_layernorm) on host arrays: out[r] = LN(x[r]) * gamma + beta over rows of 768.
void standalone_vit_layernorm(const float* x, int rows, const float* gamma, const float* beta, float* out) {
    if (rows <= 0) throw std::runtime_error("rows > 0 required");
    const size_t n = (size_t)rows * vit::D;
    float *dx = nullptr, *dg = nullptr, *db = nullptr, *dO = nullptr;
    int* dn = nullptr;
    auto cleanup = [&] { cudaFree(dx); cudaFree(dg); cudaFree(db); cudaFree(dO); cudaFree(dn); };
    try {
        RCUDA_OK(cudaMalloc(&dx, sizeof(float) * n));
        RCUDA_OK(cudaMalloc(&dO, sizeof(float) * n));
        RCUDA_OK(cudaMalloc(&dg, sizeof(float) * vit::D));
        RCUDA_OK(cudaMalloc(&db, sizeof(float) * vit::D));
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dx, x, sizeof(float) * n, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dg, gamma, sizeof(float) * vit::D, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(db, beta, sizeof(float) * vit::D, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dn, &rows, sizeof(int), cudaMemcpyHostToDevice));
        ReidModel fake;
        Launcher L{&fake, dn, 0, rows, rows, nullptr};
        L.vit_layernorm(false, dx, nullptr, dg, db, 1, dO);
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * n, cudaMemcpyDeviceToHost));
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

// Standalone attention (vit::k_vit_attention) on host arrays: qkv [n][tokens][3 * width] (q already scaled by 1/8)
// -> out [n][tokens][width]; width 768 (CLIP, 12 heads, at most 288 tokens) or 192 (ViT-Nano / ViT-Tiny, 3 heads, at
// most 320 tokens).
void standalone_vit_attention(const float* qkv, int n, int tokens, float* out, int width) {
    const int max_t = width == vit::D ? vit::MAX_T : vits::MAX_T;
    if (n <= 0 || tokens < 1 || (width != vit::D && width != vits::D) || tokens > max_t)
        throw std::runtime_error("n > 0, width 768 (1 <= tokens <= 288) or 192 (1 <= tokens <= 320) required");
    const size_t nin = (size_t)n * tokens * 3 * width, nout = (size_t)n * tokens * width;
    float *dq = nullptr, *dO = nullptr;
    int* dn = nullptr;
    auto cleanup = [&] { cudaFree(dq); cudaFree(dO); cudaFree(dn); };
    try {
        RCUDA_OK(cudaMalloc(&dq, sizeof(float) * nin));
        RCUDA_OK(cudaMalloc(&dO, sizeof(float) * nout));
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dq, qkv, sizeof(float) * nin, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dn, &n, sizeof(int), cudaMemcpyHostToDevice));
        ReidModel fake;
        Launcher L{&fake, dn, 0, n, n, nullptr};
        L.vit_attention(dq, tokens, dO, width);
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * nout, cudaMemcpyDeviceToHost));
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

namespace {
// device copies of host arrays for the standalone entry points, freed together
struct DevArrays {
    std::vector<void*> p;
    ~DevArrays() { for (void* q : p) cudaFree(q); }
    template <typename T>
    T* up(const T* host, size_t n) {
        T* d = nullptr;
        RCUDA_OK(cudaMalloc(&d, sizeof(T) * (n ? n : 1)));
        p.push_back(d);
        if (host && n) RCUDA_OK(cudaMemcpy(d, host, sizeof(T) * n, cudaMemcpyHostToDevice));
        return d;
    }
};
}  // namespace

// Standalone ViT-Nano / ViT-Tiny LayerNorm (vits::k_vits_layernorm) on host arrays: rows of 192.
void standalone_vits_layernorm(const float* x, int rows, const float* gamma, const float* beta, float* out) {
    if (rows <= 0) throw std::runtime_error("rows > 0 required");
    const size_t n = (size_t)rows * vits::D;
    DevArrays d;
    float *dx = d.up(x, n), *dg = d.up(gamma, vits::D), *db = d.up(beta, vits::D), *dO = d.up<float>(nullptr, n);
    int* dn = d.up(&rows, 1);
    ReidModel fake;
    Launcher L{&fake, dn, 0, rows, rows, nullptr};
    L.vits_layernorm(dx, dg, db, 1, dO);
    RCUDA_OK(cudaGetLastError());
    RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * n, cudaMemcpyDeviceToHost));
}

// Standalone AdaptiveINLN (vits::k_vits_ain) on host arrays: x [n][tokens][192] -> a IN(x) + b LN(x) + s.
void standalone_vits_ain(const float* x, int n, int tokens, const float* a, const float* b, const float* s,
                         float* out) {
    if (n <= 0 || tokens < 1 || vits::ain_smem_bytes(tokens) > 200 * 1024)
        throw std::runtime_error("n > 0 and 1 <= tokens <= 266 required");
    const size_t nx = (size_t)n * tokens * vits::D;
    DevArrays d;
    float *dx = d.up(x, nx), *da = d.up(a, vits::D), *db = d.up(b, vits::D), *ds = d.up(s, vits::D);
    float* dO = d.up<float>(nullptr, nx);
    int* dn = d.up(&n, 1);
    ReidModel fake;
    Launcher L{&fake, dn, 0, n, n, nullptr};
    L.vits_ain(dx, da, db, ds, tokens, dO);
    RCUDA_OK(cudaGetLastError());
    RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * nx, cudaMemcpyDeviceToHost));
}

// Standalone ViT-Nano / ViT-Tiny head (vits::k_vits_head) on host arrays: x [n][1 + gh gw][192] (the final norm's
// output), hw the head weights of weights.fold_vit for `pool` / `proj` -> out [n][feat], L2-normalised when
// `normalise`, else the row before the norm.
void standalone_vits_head(const float* x, int n, int gh, int gw, int pool, int proj, const float* hw, int n_hw,
                          int normalise, float* out) {
    const bool ok = n > 0 && gh > 0 && gw > 0 && 1 + gh * gw <= vits::MAX_T && (proj == 0 || proj == vits::PROJ) &&
                    pool >= 0 && pool <= vits::MAX_PARTS && (pool != 1 || proj == 0) && (pool < 2 || (proj && pool <= gh));
    if (!ok || (size_t)n_hw != vits::head_floats(pool, proj))
        throw std::runtime_error("n > 0, at most 320 tokens, pool 0 / 1 (no projection) / 2-3 (512-d projection) and "
                                 "the head's weight count required");
    const int T = 1 + gh * gw, feat = vits::head_feat(pool, proj);
    DevArrays d;
    float *dx = d.up(x, (size_t)n * T * vits::D), *dw = d.up(hw, (size_t)n_hw);
    float* dO = d.up<float>(nullptr, (size_t)n * feat);
    std::vector<CropDesc> crops(n);
    for (int i = 0; i < n; ++i) { std::memset(&crops[i], 0, sizeof(CropDesc)); crops[i].out_row = i; }
    CropDesc* dc = d.up(crops.data(), crops.size());
    int* dn = d.up(&n, 1);
    ReidModel fake;
    Launcher L{&fake, dn, 0, n, n, nullptr};
    L.vits_head(dx, T, gh, gw, pool, proj, dw, dc, dO, feat, normalise ? nullptr : dO);
    RCUDA_OK(cudaGetLastError());
    RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * n * feat, cudaMemcpyDeviceToHost));
}

// Standalone MLFN grouped 3x3 (mlfn::k_group_conv) on host arrays: in (n,h,w,c) NHWC, w [9][gw][c], bias [c],
// gates (n,32) -> out (n,Ho,Wo,c) = relu(conv + bias) * gates[n][channel / gw].
void standalone_mlfn_group_conv(const float* in, int n, int h, int w, int c, int gw, int stride, const float* weight,
                                const float* bias, const float* gates, float* out) {
    const int Ho = h > 0 && stride > 0 ? (h - 1) / stride + 1 : 0, Wo = w > 0 && stride > 0 ? (w - 1) / stride + 1 : 0;
    if (n <= 0 || h <= 0 || w <= 0 || (stride != 1 && stride != 2) || Wo % 4 || (gw != 4 && gw != 8 && gw != 16 && gw != 32) ||
        c != gw * mlfn::GROUPS)
        throw std::runtime_error("n, h, w > 0, stride 1 or 2, output width a multiple of 4, gw in {4, 8, 16, 32} and "
                                 "c = 32 gw required");
    const size_t n_in = (size_t)n * h * w * c, n_out = (size_t)n * Ho * Wo * c, n_w = (size_t)9 * gw * c;
    float *dx = nullptr, *dw = nullptr, *db = nullptr, *dg = nullptr, *dO = nullptr;
    int* dn = nullptr;
    auto cleanup = [&] { cudaFree(dx); cudaFree(dw); cudaFree(db); cudaFree(dg); cudaFree(dO); cudaFree(dn); };
    try {
        std::vector<float> g((size_t)n * mlfn::SHAT, 0.f);   // the kernel reads gate rows of s_hat's width
        for (int i = 0; i < n; ++i) std::memcpy(&g[(size_t)i * mlfn::SHAT], gates + (size_t)i * mlfn::GROUPS, sizeof(float) * mlfn::GROUPS);
        RCUDA_OK(cudaMalloc(&dx, sizeof(float) * n_in));
        RCUDA_OK(cudaMalloc(&dw, sizeof(float) * n_w));
        RCUDA_OK(cudaMalloc(&db, sizeof(float) * c));
        RCUDA_OK(cudaMalloc(&dg, sizeof(float) * g.size()));
        RCUDA_OK(cudaMalloc(&dO, sizeof(float) * n_out));
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dx, in, sizeof(float) * n_in, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dw, weight, sizeof(float) * n_w, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(db, bias, sizeof(float) * c, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dg, g.data(), sizeof(float) * g.size(), cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(dn, &n, sizeof(int), cudaMemcpyHostToDevice));
        ReidModel fake;
        Launcher L{&fake, dn, 0, n, n, nullptr};
        L.group_conv(dx, h, w, c, gw, stride, dw, db, dg, dO);
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaMemcpy(out, dO, sizeof(float) * n_out, cudaMemcpyDeviceToHost));
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

// Standalone MLFN factor-selection module on host arrays, as run_mlfn_chunk launches it: x (n,h,w,c) NHWC ->
// out (n,32) = sigmoid(relu(relu(GAP(x) w1 + b1) w2 + b2) w3 + b3), w1 [c][f0], w2 [f0][f1], w3 [f1][32] K-major.
void standalone_mlfn_fsm(const float* x, int n, int h, int w, int c, const float* w1, const float* b1, int f0,
                         const float* w2, const float* b2, int f1, const float* w3, const float* b3, float* out) {
    if (n <= 0 || h <= 0 || w <= 0 || c <= 0 || c % 64 || f0 <= 0 || f0 % 64 || f1 <= 0 || f1 % 64)
        throw std::runtime_error("n, h, w > 0 and c, f0, f1 positive multiples of 64 required");
    const size_t n_x = (size_t)n * h * w * c;
    std::vector<float*> bufs;
    int* dn = nullptr;
    auto cleanup = [&] { for (float* p : bufs) cudaFree(p); cudaFree(dn); };
    auto upload = [&](const float* src, size_t count) {
        float* d = nullptr;
        RCUDA_OK(cudaMalloc(&d, sizeof(float) * count));
        bufs.push_back(d);
        if (src) RCUDA_OK(cudaMemcpy(d, src, sizeof(float) * count, cudaMemcpyHostToDevice));
        return d;
    };
    try {
        std::vector<float> p1(2 * (size_t)c * f0), p2(2 * (size_t)f0 * f1);
        rn::pack_conv_weights(w1, c, f0, p1.data());
        rn::pack_conv_weights(w2, f0, f1, p2.data());
        float* dx = upload(x, n_x);
        float* dp1 = upload(p1.data(), p1.size());
        float* db1 = upload(b1, f0);
        float* dp2 = upload(p2.data(), p2.size());
        float* db2 = upload(b2, f1);
        float* dw3 = upload(w3, (size_t)f1 * mlfn::GROUPS);
        float* db3 = upload(b3, mlfn::GROUPS);
        float* pooled = upload(nullptr, (size_t)n * c);
        float* h1 = upload(nullptr, (size_t)n * f0);
        float* h2 = upload(nullptr, (size_t)n * f1);
        float* s_hat = upload(nullptr, (size_t)n * mlfn::SHAT);
        RCUDA_OK(cudaMalloc(&dn, sizeof(int)));
        RCUDA_OK(cudaMemcpy(dn, &n, sizeof(int), cudaMemcpyHostToDevice));
        ReidModel fake;
        Launcher L{&fake, dn, 0, n, n, nullptr};
        auto dense = [&](const float* in, int K, const float* pw, const float* b, int N, float* o) {
            rn::ConvArgs a{};
            a.in0 = in; a.H0 = 1; a.W0 = 1; a.C0 = K; a.k0 = 1; a.s0 = 1;
            a.w = pw; a.bias = b; a.out = o; a.Ho = 1; a.Wo = 1; a.N = N; a.relu = 1;
            L.conv_tc(a);
        };
        L.mlfn_gap(dx, h * w, c, pooled);
        dense(pooled, c, dp1, db1, f0, h1);
        dense(h1, f0, dp2, db2, f1, h2);
        L.mlfn_gate(h2, f1, dw3, db3, s_hat, 0);
        RCUDA_OK(cudaGetLastError());
        std::vector<float> s((size_t)n * mlfn::SHAT);
        RCUDA_OK(cudaMemcpy(s.data(), s_hat, sizeof(float) * s.size(), cudaMemcpyDeviceToHost));
        for (int i = 0; i < n; ++i) std::memcpy(out + (size_t)i * mlfn::GROUPS, &s[(size_t)i * mlfn::SHAT], sizeof(float) * mlfn::GROUPS);
    } catch (...) {
        cleanup();
        throw;
    }
    cleanup();
}

// ---- float32 CUDA-core kernels of the OSNet family, MobileNetV2 and LMBN_n on their own (parity tests) ----------------
// Each entry runs one kernel family through the Launcher method a loaded model calls, on a default-constructed
// ReidModel (so the template instance is the one a shipped model gets), over a crop window: the host arrays hold
// n crops, the device crop count is `count` and the chunk starts at crop `off`, so the kernels see
// clamp(count - off, 0, n) crops (chunk_count).  Every output array is uploaded as given and read back whole, so
// the caller's canaries after each tensor and in the crops outside the window come back untouched unless a kernel
// writes there.
namespace {
struct StandaloneRun {
    std::vector<void*> bufs;
    int* dn = nullptr;
    ReidModel fake;
    Launcher L;
    StandaloneRun(int n, int off, int count) : L{&fake, nullptr, off, n, n, nullptr} {
        if (n <= 0 || off < 0 || count < 0) throw std::runtime_error("n > 0, off >= 0 and count >= 0 required");
        dn = up(&count, 1);
        L.d_n = dn;
    }
    ~StandaloneRun() {
        for (void* p : bufs) cudaFree(p);
    }
    template <typename T>
    T* up(const T* src, size_t count) {
        if (!src) return nullptr;
        T* d = nullptr;
        RCUDA_OK(cudaMalloc(&d, sizeof(T) * std::max<size_t>(count, 1)));
        bufs.push_back(d);
        RCUDA_OK(cudaMemcpy(d, src, sizeof(T) * count, cudaMemcpyHostToDevice));
        return d;
    }
    void down(float* dst, const float* src, size_t count) {
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaMemcpy(dst, src, sizeof(float) * count, cudaMemcpyDeviceToHost));
    }
    // crop descriptors whose out_row fields are rows[0 .. n_rows)
    const CropDesc* crops(const int* rows, int n_rows) {
        std::vector<CropDesc> cd((size_t)n_rows);
        for (int i = 0; i < n_rows; ++i) cd[i] = CropDesc{0.f, 0.f, 0.f, 0.f, 0, rows[i]};
        return up(cd.data(), cd.size());
    }
    void report(int* instance) {
        if (instance) std::memcpy(instance, L.inst, sizeof(L.inst));
    }
};
void need(bool ok, const char* what) {
    if (!ok) throw std::runtime_error(what);
}
}  // namespace

// 1x1 GEMM (k_pointwise2): out [n][hw][nout] = act(A W + bias (+ residual)).  branches (4 x [n][hw][mid]) selects the
// gated prologue, A[m][k] = sum_b gates[crop][b][k] branch_b[m][k] for k < mid and a[m][k - mid] (downsample rows
// [n][hw][k - mid], null when k == mid) above; otherwise a is [n][hw][k].  instance: {BN, threads, gated, 0}.
void standalone_f32_pointwise(const float* a, const float* branches, const float* gates, int n, int hw, int k, int mid,
                              const float* w, int nout, const float* bias, const float* residual, int relu, int off,
                              int count, float* out, int out_floats, int* instance) {
    const bool gated = branches != nullptr;
    need(hw > 0 && k > 0 && nout > 0 && k % 4 == 0 && nout % 4 == 0 && relu >= 0 && relu <= 2 &&
             (!gated || (gates && mid > 0 && mid % 4 == 0 && mid <= k)) && (a || (gated && k == mid)) &&
             out_floats >= n * hw * nout,
         "hw, k, nout > 0, k and nout multiples of 4, relu 0-2, gated: 0 < mid <= k, mid a multiple of 4; out large enough");
    StandaloneRun r(n, off, count);
    const size_t M = (size_t)n * hw;
    PwArgs p{};
    if (gated) {
        p.in = r.up(a, M * (k - mid));
        const float* br = r.up(branches, 4 * M * mid);
        for (int b = 0; b < 4; ++b) p.branch[b] = br + b * M * mid;
        p.gates = r.up(gates, (size_t)n * 4 * mid);
        p.mid = mid;
    } else {
        p.in = r.up(a, M * k);
    }
    p.w = r.up(w, (size_t)k * nout);
    p.bias = r.up(bias, nout);
    p.residual = r.up(residual, M * nout);
    float* d_out = r.up(out, out_floats);
    p.out = d_out;
    p.K = k; p.N = nout; p.HW = hw; p.relu = relu;
    r.L.pointwise(p);
    r.down(out, d_out, out_floats);
    r.report(instance);
}

// One LightConv3x3 level of nb branches (k_lightconv2 or the generic k_lightconv), tile rows picked as run_osblock
// picks them: in nb x [n][H][W][C], wpw nb x [C][C] (K-major), wdw nb x [9][C], bias nb x [C].  Branch b writes out
// + b * out_stride ([n][H][W][C]) and, when sums is given, its per-tile channel sums to sums + b * sums_stride
// ([n][H / R][C]).  instance: {kind (1 k_lightconv, 2 k_lightconv2), C, W, R}.
void standalone_f32_lightconv(const float* in, int nb, int n, int H, int W, int C, const float* wpw, const float* wdw,
                              const float* bias, int off, int count, float* out, int out_stride, float* sums,
                              int sums_stride, int* instance) {
    need(nb >= 1 && nb <= 4 && H > 0 && W > 0 && C >= 8 && C % 8 == 0 && out_stride >= n * H * W * C &&
             out_stride % 4 == 0 && (!sums || (sums_stride >= n * H * C && sums_stride % 4 == 0)),
         "1 <= nb <= 4, H, W > 0, C a positive multiple of 8; out_stride >= n H W C, sums_stride >= n H C, both "
         "multiples of 4 (float4 stores)");
    StandaloneRun r(n, off, count);
    const size_t map = (size_t)n * H * W * C;
    const float* d_in = r.up(in, nb * map);
    const float* d_pw = r.up(wpw, (size_t)nb * C * C);
    const float* d_dw = r.up(wdw, (size_t)nb * 9 * C);
    const float* d_b = r.up(bias, (size_t)nb * C);
    float* d_out = r.up(out, (size_t)nb * out_stride);
    float* d_sums = r.up(sums, (size_t)nb * sums_stride);
    LightArgs la{};
    la.H = H; la.W = W; la.C = C; la.R = pick_tile_rows2(H, W, C);
    for (int b = 0; b < nb; ++b) {
        la.in[b] = d_in + b * map;
        la.out[b] = d_out + (size_t)b * out_stride;
        la.wpw[b] = d_pw + (size_t)b * C * C;
        la.wdw[b] = d_dw + (size_t)b * 9 * C;
        la.bias[b] = d_b + (size_t)b * C;
        la.sums[b] = d_sums ? d_sums + (size_t)b * sums_stride : nullptr;
    }
    r.L.light(la, nb, (256 / (C / 4)) * (C / 4));
    r.down(out, d_out, (size_t)nb * out_stride);
    if (sums) r.down(sums, d_sums, (size_t)nb * sums_stride);
    r.report(instance);
}

// The four LightConv branches of an OSBlock as whole-branch CTAs (k_lightchain): in [n][H][W][C] (the conv1 output),
// per LightConv l (branch b, level v: l = b (b + 1) / 2 + v - 1) wpw [10][C][C], wdw [10][9][C], bias [10][C].  Branch b
// writes out + b * out_stride and its per-tile channel sums to sums + b * sums_stride ([n][H / R][C]).  Shapes the
// model does not chain are an error.  instance: {3, C, W, R}.
void standalone_f32_lightchain(const float* in, int n, int H, int W, int C, const float* wpw, const float* wdw,
                               const float* bias, int off, int count, float* out, int out_stride, float* sums,
                               int sums_stride, int* instance) {
    need(H > 0 && W > 0 && C > 0 && out_stride >= n * H * W * C && sums_stride >= n * H * C && out_stride % 4 == 0 &&
             sums_stride % 4 == 0,
         "H, W, C > 0, out_stride >= n H W C and sums_stride >= n H C, both multiples of 4 (float4 stores), required");
    StandaloneRun r(n, off, count);
    const float* d_in = r.up(in, (size_t)n * H * W * C);
    const float* d_pw = r.up(wpw, (size_t)10 * C * C);
    const float* d_dw = r.up(wdw, (size_t)10 * 9 * C);
    const float* d_b = r.up(bias, (size_t)10 * C);
    float* d_out = r.up(out, (size_t)4 * out_stride);
    float* d_sums = r.up(sums, (size_t)4 * sums_stride);
    ChainArgs ca{};
    ca.in = d_in; ca.H = H;
    for (int b = 0; b < 4; ++b) { ca.out[b] = d_out + (size_t)b * out_stride; ca.sums[b] = d_sums + (size_t)b * sums_stride; }
    for (int l = 0; l < 10; ++l) {
        ca.wpw[l] = d_pw + (size_t)l * C * C; ca.wdw[l] = d_dw + (size_t)l * 9 * C; ca.bias[l] = d_b + (size_t)l * C;
    }
    need(r.L.light_chain(ca, C, W) > 0, "no LightConv chain kernel for this (C, W)");
    r.down(out, d_out, (size_t)4 * out_stride);
    r.down(sums, d_sums, (size_t)4 * sums_stride);
    r.report(instance);
}

// ChannelGate of an OSBlock (k_gates): sums 4 x [n][tiles][C] (branch b at b * n * tiles * C), w1 [C][hid], b1 [hid],
// w2 [hid][C], b2 [C] -> gates [n][4][C] = sigmoid(relu(mean w1 + b1) w2 + b2), mean = (sum over tiles) / hw.
void standalone_f32_gates(const float* sums, int n, int tiles, int C, int hid, int hw, const float* w1, const float* b1,
                          const float* w2, const float* b2, int off, int count, float* gates, int gates_floats) {
    need(tiles > 0 && C > 0 && hid > 0 && hw > 0 && gates_floats >= n * 4 * C,
         "tiles, C, hid, hw > 0 and gates_floats >= 4 n C required");
    StandaloneRun r(n, off, count);
    const size_t per = (size_t)n * tiles * C;
    const float* d_s = r.up(sums, 4 * per);
    float* d_g = r.up(gates, gates_floats);
    GateArgs ga{};
    for (int b = 0; b < 4; ++b) ga.sums[b] = d_s + b * per;
    ga.w1 = r.up(w1, (size_t)C * hid); ga.b1 = r.up(b1, hid); ga.w2 = r.up(w2, (size_t)hid * C); ga.b2 = r.up(b2, C);
    ga.gates = d_g; ga.C = C; ga.hid = hid; ga.tiles = tiles; ga.HW = hw;
    r.L.gates(ga);
    r.down(gates, d_g, gates_floats);
}

// Head (k_head): x [n][hw][C] -> average pool, fc + ReLU when wfc ([C][feat]) is given (else feat == C and the pooled
// row is the embedding), L2 normalisation, into row rows[off + i] of out (out_ld floats per row) for window crop i.
// rows holds off + n entries.
void standalone_f32_head(const float* x, int n, int hw, int C, const float* wfc, const float* bfc, int feat,
                         const int* rows, int off, int count, float* out, int out_floats, int out_ld) {
    need(hw > 0 && C > 0 && feat > 0 && (wfc ? bfc != nullptr : feat == C) && out_ld >= feat,
         "hw, C, feat > 0, a bias with the fc (feat == C without), out_ld >= feat required");
    for (int i = 0; i < off + n; ++i)
        need(rows[i] >= 0 && (size_t)rows[i] * out_ld + feat <= (size_t)out_floats, "an output row lies outside out");
    StandaloneRun r(n, off, count);
    const float* d_x = r.up(x, (size_t)n * hw * C);
    const float* d_w = r.up(wfc, (size_t)C * feat);
    const float* d_b = r.up(bfc, wfc ? feat : 0);
    const CropDesc* d_c = r.crops(rows, off + n);
    float* d_out = r.up(out, out_floats);
    r.L.head(d_x, hw, C, d_w, d_b, feat, d_c, d_out, out_ld);
    r.down(out, d_out, out_floats);
}

// Stems, pools and the MobileNetV2 depthwise convolution, NHWC float32, `in` [n][h][w][c_in]:
//   op 0 k_stem<false>  7x7/2 conv + bias + ReLU, in [n][h][128][3] (h 256 or 384), weight [147][c], out [n][h/2][64][c]
//   op 1 k_stem<true>   the same convolution without bias and ReLU (the instance-norm stem)
//   op 2 k_maxpool3s2   3x3/2 pad 1 max, out [n][h/2][w/2][c]
//   op 3 k_avgpool2     2x2/2 average, out [n][h/2][w/2][c]
//   op 4 k_stem3        3x3/2 pad 1 conv + bias + ReLU6, in [n][256][128][3], weight [27][c], out [n][128][64][c]
//   op 5 k_dwconv3      depthwise 3x3 pad 1 at `stride` + bias + ReLU6, weight [9][c], out [n][h/s][w/s][c]
void standalone_f32_map(int op, const float* in, int n, int h, int w, int c, int stride, const float* weight,
                        const float* bias, int off, int count, float* out, int out_floats) {
    need(op >= 0 && op <= 5 && h > 0 && w > 0 && c > 0 && c % 4 == 0, "op 0-5, h, w > 0, c a multiple of 4 required");
    if (op <= 1) need(w == IN_W && (h == IN_H || h == IN_H_MAX) && c % 16 == 0, "stem: 256 or 384 x 128 crops, c % 16 == 0");
    if (op == 4) need(w == IN_W && h == IN_H, "MobileNetV2 stem: 256 x 128 crops");
    if (op == 2 || op == 3) need(h % 2 == 0 && w % 2 == 0, "pools: even h and w");
    if (op == 5) need((stride == 1 || stride == 2) && h % stride == 0 && w % stride == 0, "depthwise: stride 1 or 2 dividing h, w");
    const int cin = (op <= 1 || op == 4) ? 3 : c;
    const int oh = op == 5 ? h / stride : h / 2, ow = op == 5 ? w / stride : (op <= 1 ? 64 : w / 2);
    need(out_floats >= n * oh * ow * c, "out too small");
    const size_t wk = op <= 1 ? 147 : (op == 4 ? 27 : 9);
    StandaloneRun r(n, off, count);
    const float* d_in = r.up(in, (size_t)n * h * w * cin);
    const float* d_w = (op == 2 || op == 3) ? nullptr : r.up(weight, wk * c);
    const float* d_b = (op == 0 || op == 4 || op == 5) ? r.up(bias, c) : nullptr;
    float* d_out = r.up(out, out_floats);
    switch (op) {
        case 0:
        case 1: r.L.stem(op == 1, d_in, d_w, d_b, c, d_out, h); break;
        case 2: r.L.maxpool(d_in, h, w, c, d_out); break;
        case 3: r.L.avgpool(d_in, h, w, c, d_out); break;
        case 4: r.L.stem3(d_in, d_w, d_b, c, d_out); break;
        case 5: r.L.dwconv3(d_in, h, w, c, stride, d_w, d_b, d_out); break;
    }
    r.down(out, d_out, out_floats);
}

// LMBN_n head: k_lmbn_pool of the bottleneck, partial and channel branch maps (x [3][n][h][w][512]) into pooled
// ([n][6][512], read back), the neck GEMMs (neck = the five reduction matrices [5][512][512], their biases [5][512],
// shared [256][512], its bias [512], reduction_ch scale / shift [4][512], concatenated in that order) and the L2
// normalisation of the 3584-d rows, written to row rows[off + i] of out as run_lmbn_chunk does.
void standalone_f32_lmbn_head(const float* x, int n, int h, int w, const float* neck, const int* rows, int off, int count,
                              float* pooled, int pooled_floats, float* out, int out_floats, int out_ld) {
    constexpr int C = LMBN_C;
    need(h > 0 && h % 2 == 0 && w > 0 && pooled_floats >= n * LMBN_POOLS * C && out_ld >= LMBN_VECS * C,
         "h even, w > 0, pooled_floats >= 6 n 512, out_ld >= 3584 required");
    for (int i = 0; i < off + n; ++i)
        need(rows[i] >= 0 && (size_t)rows[i] * out_ld + LMBN_VECS * C <= (size_t)out_floats, "an output row lies outside out");
    StandaloneRun r(n, off, count);
    const size_t map = (size_t)n * h * w * C;
    const float* d_x = r.up(x, 3 * map);
    const float* d_neck = r.up(neck, (size_t)5 * C * C + 5 * C + (size_t)(C / 2) * C + C + 4 * C);
    float* d_p = r.up(pooled, pooled_floats);
    float* d_out = r.up(out, out_floats);
    const CropDesc* d_c = r.crops(rows, off + n);
    NeckArgs na{};
    const float* q = d_neck;
    for (int k = 0; k < 5; ++k) { na.w[k] = q; q += (size_t)C * C; }
    for (int k = 0; k < 5; ++k) { na.b[k] = q; q += C; }
    na.wsh = q; q += (size_t)(C / 2) * C;
    na.bsh = q; q += C;
    na.chst = q;
    for (int which = 0; which < 3; ++which) r.L.lmbn_pool(d_x + which * map, h, w, which, d_p);
    r.L.lmbn_neck(na, d_p, d_c, d_out, out_ld);
    r.L.l2_normalise(d_c, d_out, out_ld, LMBN_VECS * C);
    r.down(pooled, d_p, pooled_floats);
    r.down(out, d_out, out_floats);
}

// ---- HACNN kernels on their own (parity tests), with the crop window and whole-array round trip described above ----
// One ConvBlock on k_conv_tc's SLICE instances: in (n,h,w,c0), weight (k*k*c0, N) K-major, out (n,Ho,Wo,out_ld) with
// columns out_off .. out_off + N - 1 = relu(conv(in) + bias); the other columns come back as given.
void standalone_hacnn_conv(const float* in, int n, int off, int count, int h, int w, int c0, int k, int stride,
                           const float* weight, int N, const float* bias, float* out, int out_ld, int out_off) {
    need(h > 0 && w > 0 && c0 > 0 && c0 % rn::KC == 0 && (k == 1 || k == 3) && (stride == 1 || stride == 2) && N > 0 &&
             N % 32 == 0 && out_off >= 0 && out_off % 2 == 0 && out_ld % 2 == 0 && out_off + N <= out_ld,
         "h, w > 0, c0 a multiple of 32, k 1 or 3, stride 1 or 2, N a multiple of 32, even out_off and out_ld, "
         "out_off + N <= out_ld required");
    StandaloneRun r(n, off, count);
    const int Ho = (h - 1) / stride + 1, Wo = (w - 1) / stride + 1, K = k * k * c0;
    std::vector<float> packed(2 * (size_t)K * N);
    rn::pack_conv_weights(weight, K, N, packed.data());
    const size_t out_floats = (size_t)n * Ho * Wo * out_ld;
    float* d_out = r.up(out, out_floats);
    rn::ConvArgs c{};
    c.in0 = r.up(in, (size_t)n * h * w * c0); c.H0 = h; c.W0 = w; c.C0 = c0; c.k0 = k; c.s0 = stride;
    c.w = r.up(packed.data(), packed.size()); c.bias = r.up(bias, N); c.out = d_out + out_off;
    c.Ho = Ho; c.Wo = Wo; c.N = N; c.relu = 1; c.out_ld = out_ld;
    r.L.conv_tc(c);
    r.down(out, d_out, out_floats);
}

// op 0: the 3x3 stride-2 stem, in (n,160,64,3), weight (27,32), bias (32) -> out (n,80,32,32);
// op 1: 3x3 stride-1 pad-1 average (/ 9), op 2: 3x3 stride-2 pad-1 max, in (n,h,w,c) -> out (n,Ho,Wo,c)
void standalone_hacnn_map(int op, const float* in, int n, int off, int count, int h, int w, int c, const float* weight,
                          const float* bias, float* out) {
    need(op >= 0 && op <= 2, "op 0 (stem), 1 (average pool) or 2 (max pool) required");
    if (op == 0) need(h == hacnn::IN_H && w == hacnn::IN_W && c == 3, "stem: 160 x 64 x 3 crops");
    else need(h > 0 && w > 0 && c > 0 && c % 4 == 0, "pools: h, w > 0 and c a multiple of 4");
    StandaloneRun r(n, off, count);
    const int s = op == 2 ? 2 : (op == 0 ? 2 : 1), co = op == 0 ? hacnn::STEM_C : c;
    const size_t out_floats = (size_t)n * ((h - 1) / s + 1) * ((w - 1) / s + 1) * co;
    const float* d_in = r.up(in, (size_t)n * h * w * c);
    float* d_out = r.up(out, out_floats);
    if (op == 0) r.L.hacnn_stem(d_in, r.up(weight, (size_t)27 * hacnn::STEM_C), r.up(bias, hacnn::STEM_C), d_out);
    else r.L.hacnn_pool(op == 2, d_in, h, w, c, d_out);
    r.down(out, d_out, out_floats);
}

// The attention of one level as run_hacnn_chunk launches it: x (n,h,w,c) -> out (n,h,w,c) = x * sigmoid(relu(
// s[p] v[o] + b[o])), s (n,h*w), v (n,c), and columns 8 level .. 8 level + 7 of theta (n,24); params holds the level's
// arrays in blob order (sp[12], w1[c][c/16], b1, w2[c/16][c], b2, wv[c][c], bv, wfc[c][8], bfc), each padded to 4.
void standalone_hacnn_attention(const float* x, int n, int off, int count, int h, int w, int c, int level,
                                const float* params, float* out, float* s, float* v, float* theta) {
    need(h > 1 && w > 1 && h % 2 == 0 && w % 2 == 0 && h * w <= hacnn::MAX_HW && c > 0 && c % 16 == 0 &&
             c <= hacnn::MAX_C && level >= 0 && level < 3,
         "even h, w > 1 with h w <= 640, c a multiple of 16 up to 384, level 0..2 required");
    StandaloneRun r(n, off, count);
    const int R = c / 16;
    const size_t sizes[9] = {12, (size_t)c * R, (size_t)R, (size_t)R * c, (size_t)c, (size_t)c * c, (size_t)c,
                             (size_t)c * 8, 8};
    size_t o[9], total = 0;
    for (int k = 0; k < 9; ++k) { o[k] = total; total += (sizes[k] + 3) / 4 * 4; }
    const float* d_p = r.up(params, total);
    const size_t nx = (size_t)n * h * w * c;
    float* d_out = r.up(out, nx);
    float* d_s = r.up(s, (size_t)n * h * w);
    float* d_v = r.up(v, (size_t)n * c);
    float* d_t = r.up(theta, (size_t)n * hacnn::THETA);
    RCUDA_OK(cudaMemcpy(d_out, x, sizeof(float) * nx, cudaMemcpyHostToDevice));   // the apply runs in place
    const hacnn::AttnW a = hacnn_attn_w(d_p, o);
    r.L.hacnn_attn(d_out, h, w, c, a, level, d_s, d_v, d_t);
    r.L.hacnn_attn_apply(d_out, h * w, c, d_s, d_v, a.bv);
    r.down(out, d_out, nx);
    r.down(s, d_s, (size_t)n * h * w);
    r.down(v, d_v, (size_t)n * c);
    r.down(theta, d_t, (size_t)n * hacnn::THETA);
}

// The STN resample of one level: src (n,H,W,C), theta (n,24) (columns 8 level .. + 7), prev (n,4,lh,lw,C) or null
// -> out (n,4,lh,lw,C)
void standalone_hacnn_stn(const float* src, int n, int off, int count, int H, int W, int C, const float* theta,
                          int level, const float* prev, int lh, int lw, float* out) {
    need(H > 1 && W > 1 && C > 0 && C % 4 == 0 && lh > 1 && lw > 1 && level >= 0 && level < 3,
         "H, W, lh, lw > 1, C a multiple of 4, level 0..2 required");
    StandaloneRun r(n, off, count);
    const size_t nl = (size_t)n * 4 * lh * lw * C;
    const float* d_t = r.up(theta, (size_t)n * hacnn::THETA);
    float* d_out = r.up(out, nl);
    r.L.hacnn_stn(r.up(src, (size_t)n * H * W * C), H, W, C, d_t + 8 * level, r.up(prev, nl), lh, lw, d_out);
    r.down(out, d_out, nl);
}

// The head: x3 (n,hw3,384) and loc (n,4,hwl,384) pooled, fc_global wg (384,512) + bg and fc_local wl (1536,512) + bl
// (K-major, BatchNorm1d folded) with ReLU into v (n,1024), then the normalised row of window crop i into out row
// rows[off + i] (rows has off + n entries; out (out_rows,1024)).
void standalone_hacnn_head(const float* x3, int n, int off, int count, int hw3, const float* loc, int hwl,
                           const float* wg, const float* bg, const float* wl, const float* bl, const int* rows,
                           int out_rows, float* out, float* v) {
    need(hw3 > 0 && hwl > 0 && out_rows > 0, "hw3, hwl, out_rows > 0 required");
    for (int i = 0; i < off + n; ++i) need(rows[i] >= 0 && rows[i] < out_rows, "rows must lie in [0, out_rows)");
    StandaloneRun r(n, off, count);
    constexpr int C = hacnn::C3, F = hacnn::HALF;
    std::vector<float> pg(2 * (size_t)C * F), pl(2 * (size_t)4 * C * F);
    rn::pack_conv_weights(wg, C, F, pg.data());
    rn::pack_conv_weights(wl, 4 * C, F, pl.data());
    float* pooled = r.up(std::vector<float>((size_t)n * 5 * C, 0.f).data(), (size_t)n * 5 * C);
    float* d_v = r.up(v, (size_t)n * hacnn::FEAT);
    float* d_out = r.up(out, (size_t)out_rows * hacnn::FEAT);
    r.L.hacnn_head_pool(r.up(x3, (size_t)n * hw3 * C), hw3, r.up(loc, (size_t)n * 4 * hwl * C), hwl, pooled,
                        pooled + (size_t)n * C);
    auto fc = [&](const float* in, int K, const float* w, const float* b, float* o) {
        rn::ConvArgs a{};
        a.in0 = in; a.H0 = 1; a.W0 = 1; a.C0 = K; a.k0 = 1; a.s0 = 1;
        a.w = w; a.bias = b; a.out = o; a.Ho = 1; a.Wo = 1; a.N = F; a.relu = 1; a.out_ld = hacnn::FEAT;
        r.L.conv_tc(a);
    };
    fc(pooled, C, r.up(pg.data(), pg.size()), r.up(bg, F), d_v);
    fc(pooled + (size_t)n * C, 4 * C, r.up(pl.data(), pl.size()), r.up(bl, F), d_v + F);
    r.L.hacnn_head(d_v, r.crops(rows, off + n), d_out, hacnn::FEAT);
    r.down(v, d_v, (size_t)n * hacnn::FEAT);
    r.down(out, d_out, (size_t)out_rows * hacnn::FEAT);
}

// ---- CSPReID-n kernels on their own (parity tests), with the crop window and whole-array round trip described above --
// One ConvBNSiLU on k_conv_tc's SILU instances: in (n,h,w,in_ld) read at channels in_off .. in_off + c0 - 1, weight
// (k*k*c0, N) K-major, residual (n,Ho,Wo,res_ld) at channels res_off .. (optional) -> out (n,Ho,Wo,out_ld) with columns
// out_off .. out_off + N - 1 = silu(conv(in) + bias) (+ residual after the activation); the other columns come back as
// given.
void standalone_cspreid_conv(const float* in, int n, int off, int count, int h, int w, int c0, int in_ld, int in_off,
                             int k, int stride, const float* weight, int N, const float* bias, const float* residual,
                             int res_ld, int res_off, float* out, int out_ld, int out_off) {
    need(h > 0 && w > 0 && c0 > 0 && (k * k * c0) % rn::KC == 0 && c0 % 4 == 0 && (k == 1 || k == 3) &&
             (stride == 1 || stride == 2) && N > 0 && N % 32 == 0 && in_off >= 0 && in_off % 4 == 0 &&
             in_ld % 4 == 0 && in_off + c0 <= in_ld && out_off >= 0 && out_off % 2 == 0 && out_ld % 2 == 0 &&
             out_off + N <= out_ld && (!residual || (res_off >= 0 && res_off % 2 == 0 && res_ld % 2 == 0 &&
                                                     res_off + N <= res_ld)),
         "h, w > 0, c0 a multiple of 4 with k k c0 a multiple of 32, k 1 or 3, stride 1 or 2, N a multiple of 32, "
         "in_off, in_ld multiples of 4 with in_off + c0 <= in_ld, even out_off / out_ld (res_off / res_ld) with "
         "out_off + N <= out_ld (res_off + N <= res_ld) required");
    StandaloneRun r(n, off, count);
    const int Ho = (h - 1) / stride + 1, Wo = (w - 1) / stride + 1, K = k * k * c0;
    std::vector<float> packed(2 * (size_t)K * N);
    rn::pack_conv_weights(weight, K, N, packed.data());
    const size_t out_floats = (size_t)n * Ho * Wo * out_ld;
    float* d_out = r.up(out, out_floats);
    rn::ConvArgs c{};
    c.in0 = r.up(in, (size_t)n * h * w * in_ld) + in_off; c.H0 = h; c.W0 = w; c.C0 = c0; c.in_ld = in_ld;
    c.k0 = k; c.s0 = stride;
    c.w = r.up(packed.data(), packed.size()); c.bias = r.up(bias, N); c.out = d_out + out_off; c.out_ld = out_ld;
    if (residual) {
        c.residual = r.up(residual, (size_t)n * Ho * Wo * res_ld) + res_off;
        c.res_ld = res_ld;
    }
    c.Ho = Ho; c.Wo = Wo; c.N = N; c.relu = residual ? 6 : 5;
    r.L.conv_tc_silu(c);
    r.down(out, d_out, out_floats);
}

// op 0: the 3x3 stride-2 stem, in (n,h,w,3), weight (27,32), bias (32) -> out (n,Ho,Wo,32) (SiLU);
// op 1: SPPF's chained 3x3 max pools, in = out (n,h,w,4c): slices 1-3 of out from slice 0 (weight, bias unused)
void standalone_cspreid_map(int op, const float* in, int n, int off, int count, int h, int w, int c,
                            const float* weight, const float* bias, float* out) {
    need(op == 0 || op == 1, "op 0 (stem) or 1 (SPPF pools) required");
    need(h > 0 && w > 0 && (op == 0 ? c == 3 : c > 0 && c % 4 == 0), "h, w > 0; the stem takes c = 3, SPPF c % 4 == 0");
    StandaloneRun r(n, off, count);
    if (op == 0) {
        const size_t out_floats = (size_t)n * ((h - 1) / 2 + 1) * ((w - 1) / 2 + 1) * csp::STEM_C;
        float* d_out = r.up(out, out_floats);
        r.L.csp_stem(r.up(in, (size_t)n * h * w * 3), h, w, r.up(weight, (size_t)27 * csp::STEM_C),
                     r.up(bias, csp::STEM_C), d_out);
        r.down(out, d_out, out_floats);
        return;
    }
    const size_t floats = (size_t)n * h * w * 4 * c;
    float* d_buf = r.up(in, floats);
    r.L.csp_sppf(d_buf, h, w, c);
    r.down(out, d_buf, floats);
}

// LightSelfAttention as run_cspreid_chunk launches it: x (n,h,w,512), h w <= 256, params in blob order (fc.0 (512,64),
// fc.2 (64,512), depthwise (9,512), depthwise shift (512), spatial 1x1 (512)) -> out (n,h,w,512)
void standalone_cspreid_attention(const float* x, int n, int off, int count, int h, int w, const float* params,
                                  float* out) {
    need(h > 0 && w > 0 && h * w <= csp::MAX_HW, "h, w > 0 with h w <= 256 required");
    StandaloneRun r(n, off, count);
    const size_t sizes[5] = {(size_t)csp::C * csp::HID, (size_t)csp::HID * csp::C, 9 * (size_t)csp::C, csp::C, csp::C};
    size_t total = 0;
    for (size_t z : sizes) total += z;
    const float* d_p = r.up(params, total);
    const float* p[5];
    for (int k = 0, o = 0; k < 5; o += (int)sizes[k], ++k) p[k] = d_p + o;
    const size_t nx = (size_t)n * h * w * csp::C;
    float* d_out = r.up(out, nx);
    r.L.csp_attn(r.up(x, nx), h, w, p, d_out);
    r.down(out, d_out, nx);
}

// The head: x (n,h,w,512), h >= 2, h w <= 256; params = bn_global, bn_part0, bn_part1 each W (512,512) K-major and b
// (512) -> row rows[off + i] of out (out_rows,1536) = the interleaved, L2-normalised row of crop i; raw (n,1536), the
// rows before the norm
void standalone_cspreid_head(const float* x, int n, int off, int count, int h, int w, const float* params,
                             const int* rows, int out_rows, float* out, float* raw) {
    need(h >= 2 && w > 0 && h * w <= csp::MAX_HW && out_rows > 0, "h >= 2, w > 0, h w <= 256, out_rows > 0 required");
    for (int i = 0; i < off + n; ++i) need(rows[i] >= 0 && rows[i] < out_rows, "rows must lie in [0, out_rows)");
    StandaloneRun r(n, off, count);
    constexpr size_t WB = (size_t)csp::C * csp::C + csp::C;
    const float* d_p = r.up(params, 3 * WB);
    const float* p[6] = {d_p, d_p + csp::C * csp::C, d_p + WB, d_p + WB + csp::C * csp::C, d_p + 2 * WB,
                         d_p + 2 * WB + csp::C * csp::C};
    float* d_raw = r.up(raw, (size_t)n * csp::FEAT);
    float* d_out = r.up(out, (size_t)out_rows * csp::FEAT);
    r.L.csp_head(r.up(x, (size_t)n * h * w * csp::C), h, w, p, r.crops(rows, off + n), d_out, csp::FEAT, d_raw);
    r.down(raw, d_raw, (size_t)n * csp::FEAT);
    r.down(out, d_out, (size_t)out_rows * csp::FEAT);
}

}  // namespace bmb
