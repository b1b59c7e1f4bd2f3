// vit_small.cuh -- the non-GEMM kernels of the ViT-Nano / ViT-Tiny ReID family (reid/backbones/vit_nano.py ViTNano and
// vit_tiny.py ViTTinyParts, eval mode): width 192, 3 heads of 64, pre-norm blocks, a final LayerNorm and a BNNeck head.
// The linear layers (patch embedding, qkv, proj, fc1 + GELU, fc2) run on rn::k_conv_tc as 1x1 convolutions over a
// [crops x tokens] x 1 map, the attention on vit::k_vit_attention<192, 320>, the patch rows on vit::k_vit_patchify.
// What is here:
//
//   k_vits_tokens     token assembly into the residual stream: row 0 the positional table's row 0 (which carries the
//                     class token), row t the patch-embedding row t - 1 plus positional row t
//   k_vits_layernorm  one warp per 192-wide token row (6 channels per lane), two-pass mean / variance, eps 1e-5
//   k_vits_ain        AdaptiveINLN of one crop per CTA, its [T][192] tile in shared memory: per-channel instance
//                     statistics over all T tokens (biased variance), per-row LayerNorm statistics, then
//                     a[c] IN(x) + b[c] LN(x) + s[c] (gate and both affines folded at export)
//   k_vits_head       CLS / CLS + proj / omni-scale / part pooling, the folded BatchNorm1d(s), the L2 norm
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vit_tc.cuh"

namespace bmb {
namespace vits {

constexpr int D = 192;           // embed dim
constexpr int HEADS = 3;
constexpr int MLP = 4 * D;       // 768
constexpr int PROJ = 512;        // proj / part_projs output
constexpr int OS_MID = 12;       // omni-scale gate hidden width (192 / 16)
constexpr int OS_SCALES = 4;
constexpr int MAX_T = 320;       // attention instance: vit_tiny's 311 tokens
constexpr int MAX_PARTS = 3;
constexpr int MAX_FEAT = (1 + MAX_PARTS) * PROJ;
constexpr int AIN_THREADS = 256;
constexpr int HEAD_THREADS = 256;
constexpr float EPS = 1e-5f;

// floats of k_vits_head's weights for a pooling mode (0 CLS, 1 omni-scale, P >= 2 parts) and projection width
__host__ __device__ inline size_t head_floats(int pool, int proj) {
    if (pool == 1) return (size_t)OS_SCALES * 2 * D + (size_t)D * OS_MID + OS_MID + (size_t)OS_MID * D + D + 2 * D;
    const int vecs = pool >= 2 ? 1 + pool : 1;
    return proj ? (size_t)vecs * ((size_t)D * proj + proj) : 2 * (size_t)D;
}
// the head row's width
__host__ __device__ inline int head_feat(int pool, int proj) {
    if (pool == 1 || !proj) return D;
    return (pool >= 2 ? 1 + pool : 1) * proj;
}

inline size_t ain_smem_bytes(int T) { return sizeof(float) * ((size_t)T * D + 2 * D); }

__device__ __forceinline__ int clamp_crops(const int* d_n, int off, int cap) {
    const int n = *d_n - off;
    return n < 0 ? 0 : (n > cap ? cap : n);
}

// patch [crops][T - 1][192], pos [T][192] -> x [crops][T][192]; one thread per float4
__global__ void k_vits_tokens(const float* __restrict__ patch, const float* __restrict__ pos, int T,
                              const int* __restrict__ d_n, int off, int cap, float* __restrict__ x) {
    const int n_crops = clamp_crops(d_n, off, cap);
    const size_t total = (size_t)n_crops * T * (D / 4);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(i % (D / 4));
        const size_t r = i / (D / 4);
        const int n = (int)(r / T), t = (int)(r - (size_t)n * T);
        float4 v = reinterpret_cast<const float4*>(pos + (size_t)t * D)[q];
        if (t > 0) {
            const float4 p = reinterpret_cast<const float4*>(patch + ((size_t)n * (T - 1) + t - 1) * D)[q];
            v = make_float4(p.x + v.x, p.y + v.y, p.z + v.z, p.w + v.w);
        }
        reinterpret_cast<float4*>(x)[i] = v;
    }
}

// out[r] = LN(x[r]) * gamma + beta over the T rows of every crop in the chunk
__global__ void __launch_bounds__(256) k_vits_layernorm(const float* __restrict__ in, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, int T,
                                                        const int* __restrict__ d_n, int off, int cap,
                                                        float* __restrict__ out) {
    const int n_crops = clamp_crops(d_n, off, cap);
    const int lane = threadIdx.x & 31;
    const size_t rows = (size_t)n_crops * T;
    for (size_t r = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; r < rows;
         r += ((size_t)gridDim.x * blockDim.x) >> 5) {
        const float* xr = in + r * D;
        float v[6];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) { v[i] = xr[lane + 32 * i]; s += v[i]; }
        const float mean = vit::warp_sum(s) * (1.f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) { const float d = v[i] - mean; q = fmaf(d, d, q); }
        const float rstd = rsqrtf(vit::warp_sum(q) * (1.f / D) + EPS);
        float* o = out + r * D;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const int c = lane + 32 * i;
            o[c] = (v[i] - mean) * rstd * gamma[c] + beta[c];
        }
    }
}

// AdaptiveINLN, one CTA per crop (grid = crops): out = a * IN(x) + b * LN(x) + s with a = sigmoid(gate) in_norm.weight,
// b = (1 - sigmoid(gate)) ln.weight, s = sigmoid(gate) in_norm.bias + (1 - sigmoid(gate)) ln.bias
__global__ void __launch_bounds__(AIN_THREADS) k_vits_ain(const float* __restrict__ x, int T,
                                                          const float* __restrict__ a, const float* __restrict__ b,
                                                          const float* __restrict__ s, const int* __restrict__ d_n,
                                                          int off, int cap, float* __restrict__ out) {
    const int n = blockIdx.x;
    if (n >= clamp_crops(d_n, off, cap)) return;
    extern __shared__ __align__(16) float tile[];   // [T][192], then the column mean and rstd
    float* cmean = tile + (size_t)T * D;
    float* crstd = cmean + D;
    const float4* src = reinterpret_cast<const float4*>(x + (size_t)n * T * D);
    for (int i = threadIdx.x; i < T * (D / 4); i += blockDim.x) reinterpret_cast<float4*>(tile)[i] = src[i];
    __syncthreads();
    for (int c = threadIdx.x; c < D; c += blockDim.x) {   // instance statistics of channel c over the T tokens
        float sum = 0.f;
        for (int t = 0; t < T; ++t) sum += tile[t * D + c];
        const float mean = sum / (float)T;
        float q = 0.f;
        for (int t = 0; t < T; ++t) { const float d = tile[t * D + c] - mean; q = fmaf(d, d, q); }
        cmean[c] = mean;
        crstd[c] = rsqrtf(q / (float)T + EPS);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* dst = out + (size_t)n * T * D;
    for (int t = warp; t < T; t += AIN_THREADS / 32) {
        float v[6];
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) { v[i] = tile[t * D + lane + 32 * i]; sum += v[i]; }
        const float mean = vit::warp_sum(sum) * (1.f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) { const float d = v[i] - mean; q = fmaf(d, d, q); }
        const float rstd = rsqrtf(vit::warp_sum(q) * (1.f / D) + EPS);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const int c = lane + 32 * i;
            dst[t * D + c] = a[c] * ((v[i] - cmean[c]) * crstd[c]) + b[c] * ((v[i] - mean) * rstd) + s[c];
        }
    }
}

// Head, one CTA per crop.  x: the final LayerNorm's output [crops][T][192] on a gh x gw patch grid.  hw: the head's
// weights (weights.fold_vit's head layout for `pool` / `proj`).  Writes the L2-normalised row to
// out + crops[off + n].out_row * out_ld, or, when `tap` is set, the un-normalised row to tap + n * feat.
__global__ void __launch_bounds__(HEAD_THREADS) k_vits_head(const float* __restrict__ x, int T, int gh, int gw,
                                                            int pool, int proj, const float* __restrict__ hw,
                                                            const CropDesc* __restrict__ crops,
                                                            const int* __restrict__ d_n, int off, int cap,
                                                            float* __restrict__ out, int out_ld,
                                                            float* __restrict__ tap) {
    const int n = blockIdx.x;
    if (n >= clamp_crops(d_n, off, cap)) return;
    __shared__ float v[1 + MAX_PARTS][D];   // pooled vectors: the class token (or the patch mean), then the parts
    __shared__ float f[MAX_FEAT];
    __shared__ float hid[OS_MID];
    __shared__ float red[HEAD_THREADS / 32 + 2];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* xb = x + (size_t)n * T * D;
    const int parts = pool >= 2 ? pool : 0;
    for (int c = tid; c < D; c += blockDim.x) {
        if (pool == 1) {   // every scale's strip pooling averages to the patch mean on a grid whose height 8 divides
            float sum = 0.f;
            for (int t = 1; t < T; ++t) sum += xb[(size_t)t * D + c];
            v[0][c] = sum / (float)(T - 1);
        } else {
            v[0][c] = xb[c];
        }
        const int sh = parts ? gh / parts : 0;
        for (int p = 0; p < parts; ++p) {   // grid rows [p sh, p sh + sh), the last strip to the bottom
            const int r0 = p * sh, r1 = p == parts - 1 ? gh : r0 + sh;
            float sum = 0.f;
            for (int r = r0; r < r1; ++r)
                for (int q = 0; q < gw; ++q) sum += xb[(size_t)(1 + r * gw + q) * D + c];
            v[1 + p][c] = sum / (float)((r1 - r0) * gw);
        }
    }
    __syncthreads();
    const int feat = head_feat(pool, proj);
    if (pool == 1) {
        // f = sum_i g_i * q_i, q_i = scale_norms[i](p), g_i = sigmoid(W2 relu(W1 q_i + b1) + b2); then the BNNeck
        if (warp == 0) {   // LayerNorm statistics of the pooled vector (the four scales differ only in the affine)
            float p[6], sum = 0.f;
#pragma unroll
            for (int i = 0; i < 6; ++i) { p[i] = v[0][lane + 32 * i]; sum += p[i]; }
            const float mean = vit::warp_sum(sum) * (1.f / D);
            float q = 0.f;
#pragma unroll
            for (int i = 0; i < 6; ++i) { const float d = p[i] - mean; q = fmaf(d, d, q); }
            const float rstd = rsqrtf(vit::warp_sum(q) * (1.f / D) + EPS);
            if (lane == 0) { red[0] = mean; red[1] = rstd; }
        }
        __syncthreads();
        const float mean = red[0], rstd = red[1];
        const float* w1 = hw + (size_t)OS_SCALES * 2 * D;
        const float* b1 = w1 + (size_t)D * OS_MID;
        const float* w2 = b1 + OS_MID;
        const float* b2 = w2 + (size_t)OS_MID * D;
        const float* bsc = b2 + D;
        const float* bsh = bsc + D;
        float fused = 0.f;
        for (int i = 0; i < OS_SCALES; ++i) {
            const float* g = hw + (size_t)i * 2 * D;
            float qc = 0.f;
            if (tid < D) {
                qc = (v[0][tid] - mean) * rstd * g[tid] + g[D + tid];
                v[1][tid] = qc;
            }
            __syncthreads();
            if (tid < OS_MID) {
                float h = b1[tid];
                for (int k = 0; k < D; ++k) h = fmaf(v[1][k], w1[k * OS_MID + tid], h);
                hid[tid] = fmaxf(h, 0.f);
            }
            __syncthreads();
            if (tid < D) {
                float z = b2[tid];
#pragma unroll
                for (int j = 0; j < OS_MID; ++j) z = fmaf(hid[j], w2[j * D + tid], z);
                fused += qc / (1.f + expf(-z));
            }
            __syncthreads();
        }
        if (tid < D) f[tid] = fused * bsc[tid] + bsh[tid];
    } else if (!proj) {   // the class token through the folded bottleneck
        for (int c = tid; c < D; c += blockDim.x) f[c] = v[0][c] * hw[c] + hw[D + c];
    } else {   // per pooled vector k: the folded proj (or part_projs[k - 1]) + BatchNorm1d
        const int vecs = 1 + parts;
        for (int o = tid; o < vecs * proj; o += blockDim.x) {
            const int k = o / proj, c = o - k * proj;
            const float* w = hw + (size_t)k * ((size_t)D * proj + proj);
            float t4[4] = {0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < D; j += 4) {
#pragma unroll
                for (int u = 0; u < 4; ++u) t4[u] = fmaf(v[k][j + u], w[(size_t)(j + u) * proj + c], t4[u]);
            }
            f[o] = w[(size_t)D * proj + c] + ((t4[0] + t4[1]) + (t4[2] + t4[3]));
        }
    }
    __syncthreads();
    if (tap) {
        for (int c = tid; c < feat; c += blockDim.x) tap[(size_t)n * feat + c] = f[c];
        return;
    }
    float sq = 0.f;
    for (int c = tid; c < feat; c += blockDim.x) sq += f[c] * f[c];
    sq = vit::warp_sum(sq);
    if (lane == 0) red[warp] = sq;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    const float nrm = sqrtf(tot);
    float* dst = out + (size_t)crops[off + n].out_row * out_ld;
    for (int c = tid; c < feat; c += blockDim.x) dst[c] = f[c] / nrm;
}

}  // namespace vits
}  // namespace bmb
