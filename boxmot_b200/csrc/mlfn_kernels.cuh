// mlfn_kernels.cuh -- the parts of an MLFN block (reid/backbones/mlfn.py) that are not dense 1x1 convolutions (those run
// on rn::k_conv_tc):
//   k_group_conv   the grouped 3x3 fm_conv2 (32 groups of width GW = 4 / 8 / 16 / 32, pad 1, stride 1 or 2) with its
//                  folded BN bias, the ReLU and the factor-selection gate of the channel's group in the epilogue.
//                  float32 FMA on the CUDA cores: a block-diagonal tensor-core GEMM would multiply 32 / GW times the
//                  real work (DESIGN.md section 3.3e).  A thread owns 4 consecutive output channels (one group) at 4
//                  consecutive output pixels of a row, so every weight float4 it loads feeds 16 FMAs; consecutive
//                  threads own consecutive channel quads of the same pixels (coalesced loads and stores).
//   k_mlfn_gap     the average pool of a block input (or of the last block's output) per crop and channel: 16 pixel
//                  stripes per 64 channels, combined in a fixed order, so a crop's row never depends on its neighbours.
//   k_mlfn_gate    the FSM's last layer (f1 -> 32) and the sigmoid, one warp per crop, written into the block's 32
//                  columns of the [crops][512] s_hat rows.
//   k_mlfn_head    v = 0.5 (x + s) (the sum comes from fc_s's RELU_RES epilogue), L2-normalised into the caller's rows.
#pragma once
#include <cuda_runtime.h>

namespace bmb {
namespace mlfn {

constexpr int GROUPS = 32;
constexpr int BLOCKS = 16;
constexpr int SHAT = GROUPS * BLOCKS;   // 512 gates per crop
constexpr int FEAT = 1024;

__device__ __forceinline__ int crops_in_chunk(const int* d_n, int off, int cap) {
    int n = *d_n - off;
    n = n < 0 ? 0 : n;
    return n > cap ? cap : n;
}

// in [crops][H][W][C] -> out [crops][Ho][Wo][C], Ho = (H - 1) / stride + 1 (likewise Wo, a multiple of 4);
// w [9][GW][C]: element (tap, i, c) weighs input channel (c / GW) GW + i; gates: row n at gates + n * gate_ld,
// column c / GW.  out = relu(conv + bias) * gate.
template <int GW>
__global__ void __launch_bounds__(256) k_group_conv(const float* __restrict__ in, int H, int W, int C, int stride,
                                                    const float* __restrict__ w, const float* __restrict__ bias,
                                                    const float* __restrict__ gates, int gate_ld,
                                                    const int* __restrict__ d_n, int off, int cap,
                                                    float* __restrict__ out) {
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
    const int cq = C / 4, xq = Wo / 4;
    const size_t items = (size_t)crops_in_chunk(d_n, off, cap) * Ho * xq * cq;
    const size_t item = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (item >= items) return;
    const int c0 = (int)(item % cq) * 4;
    size_t rest = item / cq;
    const int ox0 = (int)(rest % xq) * 4;
    rest /= xq;
    const int oy = (int)(rest % Ho);
    const int n = (int)(rest / Ho);
    const int g = c0 / GW;
    const float* src = in + (size_t)n * H * W * C + g * GW;

    float4 acc[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy * stride + ky - 1;
        if (iy < 0 || iy >= H) continue;
        const float* row = src + (size_t)iy * W * C;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const float* wt = w + (size_t)((ky * 3 + kx) * GW) * C + c0;
            int ix[4];
            bool ok[4];
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                ix[p] = (ox0 + p) * stride + kx - 1;
                ok[p] = ix[p] >= 0 && ix[p] < W;
            }
#pragma unroll
            for (int i = 0; i < GW; i += 4) {
                const float4 w0 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(i + 0) * C));
                const float4 w1 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(i + 1) * C));
                const float4 w2 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(i + 2) * C));
                const float4 w3 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(i + 3) * C));
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    const float4 a = ok[p] ? __ldg(reinterpret_cast<const float4*>(row + (size_t)ix[p] * C + i))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
                    float4& o = acc[p];
                    o.x = fmaf(a.x, w0.x, o.x); o.y = fmaf(a.x, w0.y, o.y); o.z = fmaf(a.x, w0.z, o.z); o.w = fmaf(a.x, w0.w, o.w);
                    o.x = fmaf(a.y, w1.x, o.x); o.y = fmaf(a.y, w1.y, o.y); o.z = fmaf(a.y, w1.z, o.z); o.w = fmaf(a.y, w1.w, o.w);
                    o.x = fmaf(a.z, w2.x, o.x); o.y = fmaf(a.z, w2.y, o.y); o.z = fmaf(a.z, w2.z, o.z); o.w = fmaf(a.z, w2.w, o.w);
                    o.x = fmaf(a.w, w3.x, o.x); o.y = fmaf(a.w, w3.y, o.y); o.z = fmaf(a.w, w3.z, o.z); o.w = fmaf(a.w, w3.w, o.w);
                }
            }
        }
    }
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + c0));
    const float s = gates[(size_t)n * gate_ld + g];
    float* dst = out + (((size_t)n * Ho + oy) * Wo + ox0) * C + c0;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        float4 o = acc[p];
        o.x = fmaxf(o.x + b.x, 0.f) * s; o.y = fmaxf(o.y + b.y, 0.f) * s;
        o.z = fmaxf(o.z + b.z, 0.f) * s; o.w = fmaxf(o.w + b.w, 0.f) * s;
        *reinterpret_cast<float4*>(dst + (size_t)p * C) = o;
    }
}

// x [crops][HW][C] -> out [crops][C] (mean over HW); grid (C / 64, crops), 256 threads; C a multiple of 64
__global__ void __launch_bounds__(256) k_mlfn_gap(const float* __restrict__ x, int HW, int C, const int* __restrict__ d_n,
                                                  int off, int cap, float* __restrict__ out) {
    const int n = blockIdx.y;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    __shared__ float4 part[16][16];
    const int q = threadIdx.x & 15, stripe = threadIdx.x >> 4;
    const int c = blockIdx.x * 64 + 4 * q;
    const float* src = x + (size_t)n * HW * C + c;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = stripe; p < HW; p += 16) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + (size_t)p * C));
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    part[stripe][q] = s;
    __syncthreads();
    if (threadIdx.x < 64) {
        const int qq = threadIdx.x >> 2, e = threadIdx.x & 3;
        float t = 0.f;
        for (int k = 0; k < 16; ++k) t += reinterpret_cast<const float*>(&part[k][qq])[e];
        out[(size_t)n * C + blockIdx.x * 64 + threadIdx.x] = t / (float)HW;
    }
}

// h [crops][F1] -> s_hat[n * SHAT + col + j] = sigmoid(b[j] + sum_k h[n][k] w[k][j]), j < 32; one warp per crop
__global__ void __launch_bounds__(256) k_mlfn_gate(const float* __restrict__ h, int F1, const float* __restrict__ w,
                                                   const float* __restrict__ b, const int* __restrict__ d_n, int off,
                                                   int cap, float* __restrict__ s_hat, int col) {
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5), j = threadIdx.x & 31;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    const float* hr = h + (size_t)n * F1;
    float t0 = 0.f, t1 = 0.f, t2 = 0.f, t3 = 0.f;
    for (int k = 0; k < F1; k += 4) {
        t0 = fmaf(hr[k], w[(size_t)k * GROUPS + j], t0);
        t1 = fmaf(hr[k + 1], w[(size_t)(k + 1) * GROUPS + j], t1);
        t2 = fmaf(hr[k + 2], w[(size_t)(k + 2) * GROUPS + j], t2);
        t3 = fmaf(hr[k + 3], w[(size_t)(k + 3) * GROUPS + j], t3);
    }
    const float z = b[j] + ((t0 + t1) + (t2 + t3));
    s_hat[(size_t)n * SHAT + col + j] = 1.f / (1.f + expf(-z));
}

// xs [crops][FEAT] = x + s -> v = 0.5 xs; out row crops[off + n].out_row = v / ||v||; v_tap (optional) [crops][FEAT] = v
template <typename Crop>
__global__ void __launch_bounds__(256) k_mlfn_head(const float* __restrict__ xs, const Crop* __restrict__ crops,
                                                   const int* __restrict__ d_n, int off, int cap, float* __restrict__ out,
                                                   int out_ld, float* __restrict__ v_tap) {
    const int n = blockIdx.x;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    __shared__ float red[8];
    const float* src = xs + (size_t)n * FEAT;
    float v[FEAT / 256];
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < FEAT / 256; ++k) {
        v[k] = 0.5f * src[threadIdx.x + 256 * k];
        sq = fmaf(v[k], v[k], sq);
    }
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
    __syncthreads();
    float tot = 0.f;
    for (int i = 0; i < 8; ++i) tot += red[i];
    const float nrm = sqrtf(tot);
    float* dst = out + (size_t)crops[off + n].out_row * out_ld;
#pragma unroll
    for (int k = 0; k < FEAT / 256; ++k) {
        dst[threadIdx.x + 256 * k] = v[k] / nrm;
        if (v_tap) v_tap[(size_t)n * FEAT + threadIdx.x + 256 * k] = v[k];
    }
}

}  // namespace mlfn
}  // namespace bmb
