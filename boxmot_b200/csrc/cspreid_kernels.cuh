// cspreid_kernels.cuh -- the float32 CUDA-core kernels of the CSPReID-n ReID path (reid/backbones/cspreid_n.py, eval
// mode).  Every ConvBNSiLU after the first stem conv runs on rn::k_conv_tc's SILU instances; these kernels do the rest.
// All maps are NHWC.
//   k_stem      the 3 -> 32 3x3 stride-2 ConvBNSiLU (BN folded) on the H x W crop.
//   k_sppf      SPPF's three chained MaxPool2d(3, 1, 1) in one pass: the i-th pool of a stride-1 max pool chain is the
//               max over the (2i + 1)^2 window clipped to the map (-inf padding never wins), so each output is exact.
//               Reads slice 0 of SPPF's concatenation and writes slices 1-3.
//   k_attn      LightSelfAttention, one CTA per crop: the channel gate (average pool, 1x1 C -> C/8, SiLU, 1x1 back,
//               sigmoid), then the spatial gate (depthwise 3x3 + folded BN + SiLU, 1x1 C -> 1, sigmoid) of the gated
//               map, then out = x * ca[c] * sa[p].
//   k_head      the global and the two half-height average pools (AdaptiveAvgPool2d((2, 1))), the three BNNeck3
//               GEMVs (BatchNorm1d folded), the interleaved store (element 3 c + branch) and the L2 norm.
// Reductions run in a fixed order without atomics, so a crop's row never depends on its place in a chunk.
#pragma once
#include <cuda_runtime.h>

#include "mlfn_kernels.cuh"

namespace bmb {
namespace csp {

using mlfn::crops_in_chunk;

constexpr int STEM_C = 32;
constexpr int C = 512;          // the width of stage 4, the attention and the head
constexpr int HID = 64;         // the channel gate's hidden width (C / 8)
constexpr int SPPF_C = 256;     // SPPF's hidden width: four slices of its 1024-wide concatenation
constexpr int FEAT = 3 * C;
constexpr int MAX_HW = 256;     // the largest attended / pooled map (8 x 8 at 256 x 256 crops)
constexpr int HEAD_CROPS = 4;   // crops per head CTA: each weight load feeds four crops

// blob [crops][H][W][3] -> out [crops][Ho][Wo][32], Ho = (H - 1) / 2 + 1; w [27][32] (k = (kh*3 + kw)*3 + ci), b [32];
// one thread per output pixel and channel quad
__global__ void __launch_bounds__(256) k_stem(const float* __restrict__ blob, int H, int W, const float* __restrict__ w,
                                              const float* __restrict__ b, const int* __restrict__ d_n, int off, int cap,
                                              float* __restrict__ out) {
    constexpr int CQ = STEM_C / 4;
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    const size_t items = (size_t)crops_in_chunk(d_n, off, cap) * Ho * Wo * CQ;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(it % CQ);
        const size_t px = it / CQ;
        const int ox = (int)(px % Wo), oy = (int)(px / Wo % Ho), n = (int)(px / ((size_t)Wo * Ho));
        const float* src = blob + (size_t)n * H * W * 3;
        float4 acc = __ldg(reinterpret_cast<const float4*>(b) + q);
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = 2 * oy + ky - 1;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = 2 * ox + kx - 1;
                if (ix < 0 || ix >= W) continue;
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const float a = src[((size_t)iy * W + ix) * 3 + ci];
                    const float4 wv = __ldg(reinterpret_cast<const float4*>(w + ((ky * 3 + kx) * 3 + ci) * STEM_C) + q);
                    acc.x = fmaf(a, wv.x, acc.x); acc.y = fmaf(a, wv.y, acc.y);
                    acc.z = fmaf(a, wv.z, acc.z); acc.w = fmaf(a, wv.w, acc.w);
                }
            }
        }
        acc.x /= 1.f + expf(-acc.x); acc.y /= 1.f + expf(-acc.y);
        acc.z /= 1.f + expf(-acc.z); acc.w /= 1.f + expf(-acc.w);
        reinterpret_cast<float4*>(out)[it] = acc;
    }
}

// buf [crops][H][W][4 c] (c a multiple of 4): slice i = 1..3 (channels i c .. i c + c - 1) = max of slice 0 over the
// (2i + 1) x (2i + 1) window around each pixel, clipped to the map
__global__ void __launch_bounds__(256) k_sppf(float* __restrict__ buf, int H, int W, int c, const int* __restrict__ d_n,
                                              int off, int cap) {
    const int cq = c / 4, ld = 4 * c;
    const size_t items = (size_t)crops_in_chunk(d_n, off, cap) * H * W * cq;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(it % cq);
        const size_t px = it / cq;
        const int x = (int)(px % W), y = (int)(px / W % H);
        const size_t n = px / ((size_t)W * H);
        const float* src = buf + n * H * W * ld + 4 * q;
        float4 r[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) r[i] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int dy = -3; dy <= 3; ++dy) {
            const int iy = y + dy;
            if (iy < 0 || iy >= H) continue;
            for (int dx = -3; dx <= 3; ++dx) {
                const int ix = x + dx;
                if (ix < 0 || ix >= W) continue;
                const float4 v = *reinterpret_cast<const float4*>(src + ((size_t)iy * W + ix) * ld);
                const int ring = max(abs(dy), abs(dx));   // the first pool whose window holds this tap
#pragma unroll
                for (int i = 0; i < 3; ++i)
                    if (ring <= i + 1) {
                        r[i].x = fmaxf(r[i].x, v.x); r[i].y = fmaxf(r[i].y, v.y);
                        r[i].z = fmaxf(r[i].z, v.z); r[i].w = fmaxf(r[i].w, v.w);
                    }
            }
        }
        float* dst = buf + px * ld + 4 * q;
#pragma unroll
        for (int i = 0; i < 3; ++i) *reinterpret_cast<float4*>(dst + (i + 1) * c) = r[i];
    }
}

// x [crops][H][W][512] -> out [crops][H][W][512] (H W <= MAX_HW); w1 [512][64], w2 [64][512] (K-major, no bias),
// dw [9][512] (BN scale folded), db [512] (BN shift), ws [512] (the spatial 1x1, no bias).  One CTA of 512 threads per
// crop, thread = channel.
__global__ void __launch_bounds__(C) k_attn(const float* __restrict__ x, int H, int W, const float* __restrict__ w1,
                                            const float* __restrict__ w2, const float* __restrict__ dw,
                                            const float* __restrict__ db, const float* __restrict__ ws,
                                            const int* __restrict__ d_n, int off, int cap, float* __restrict__ out) {
    const int n = blockIdx.x;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    constexpr int WARPS = C / 32;
    __shared__ float gap[C], hid[HID], part[MAX_HW][WARPS], sa[MAX_HW];
    const int HW = H * W, c = threadIdx.x, warp = c >> 5, lane = c & 31;
    const float* xs = x + (size_t)n * HW * C;
    float t = 0.f;
    for (int p = 0; p < HW; ++p) t += xs[(size_t)p * C + c];
    gap[c] = t / (float)HW;
    __syncthreads();
    for (int j = warp; j < HID; j += WARPS) {   // fc.0 + SiLU: one warp per hidden unit, lanes over channels
        float h = 0.f;
        for (int k = lane; k < C; k += 32) h = fmaf(gap[k], w1[(size_t)k * HID + j], h);
        for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
        if (lane == 0) hid[j] = h / (1.f + expf(-h));
    }
    __syncthreads();
    float g = 0.f;
    for (int j = 0; j < HID; ++j) g = fmaf(hid[j], w2[(size_t)j * C + c], g);
    const float ca = 1.f / (1.f + expf(-g));
    float wd[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wd[k] = dw[k * C + c];
    const float bc = db[c], wc = ws[c];
    for (int p = 0; p < HW; ++p) {   // depthwise 3x3 of the gated map + BN + SiLU, weighed by the spatial 1x1
        const int y = p / W, xx = p - y * W;
        float d = bc;
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            const int iy = y + k / 3 - 1, ix = xx + k % 3 - 1;
            if (iy >= 0 && iy < H && ix >= 0 && ix < W) d = fmaf(wd[k], xs[((size_t)iy * W + ix) * C + c] * ca, d);
        }
        float v = wc * (d / (1.f + expf(-d)));
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) part[p][warp] = v;
    }
    __syncthreads();
    for (int p = c; p < HW; p += C) {
        float s = 0.f;
        for (int k = 0; k < WARPS; ++k) s += part[p][k];
        sa[p] = 1.f / (1.f + expf(-s));
    }
    __syncthreads();
    float* os = out + (size_t)n * HW * C;
    for (int p = 0; p < HW; ++p) os[(size_t)p * C + c] = (xs[(size_t)p * C + c] * ca) * sa[p];
}

// x [crops][H][W][512] (H >= 2, H W <= MAX_HW) -> row crops[off + n].out_row of out: element 3 c + b of the
// [global | part 0 | part 1] BNNeck3 outputs v_b = W_b^T pool_b + bias_b (W_b [512][512] K-major, BatchNorm1d folded),
// divided by the row's L2 norm.  Part i pools rows floor(i H / 2) .. ceil((i + 1) H / 2) - 1 (AdaptiveAvgPool2d).
// raw, when non-null, receives the row before the norm at raw + n * FEAT.  One CTA of 512 threads per HEAD_CROPS crops.
template <typename Crop>
__global__ void __launch_bounds__(C) k_head(const float* __restrict__ x, int H, int W, const float* __restrict__ wg,
                                            const float* __restrict__ bg, const float* __restrict__ w0,
                                            const float* __restrict__ b0, const float* __restrict__ w1,
                                            const float* __restrict__ b1, const Crop* __restrict__ crops,
                                            const int* __restrict__ d_n, int off, int cap, float* __restrict__ out,
                                            int out_ld, float* __restrict__ raw) {
    const int count = crops_in_chunk(d_n, off, cap);
    const int n0 = blockIdx.x * HEAD_CROPS;
    if (n0 >= count) return;
    const int nc = min(HEAD_CROPS, count - n0);
    constexpr int WARPS = C / 32;
    __shared__ float pool[HEAD_CROPS][3][C], red[HEAD_CROPS][WARPS];
    const int c = threadIdx.x, warp = c >> 5, lane = c & 31, HW = H * W;
    const int e0 = (H + 1) / 2, s1 = H / 2;   // part 0: rows 0 .. e0 - 1, part 1: rows s1 .. H - 1
    for (int j = 0; j < HEAD_CROPS; ++j) {
        float t0 = 0.f, t1 = 0.f, t = 0.f;
        if (j < nc) {
            const float* xs = x + (size_t)(n0 + j) * HW * C + c;
            for (int y = 0; y < H; ++y) {
                float r = 0.f;
                for (int xx = 0; xx < W; ++xx) r += xs[((size_t)y * W + xx) * C];
                t += r;
                if (y < e0) t0 += r;
                if (y >= s1) t1 += r;
            }
        }
        pool[j][0][c] = t / (float)HW;
        pool[j][1][c] = t0 / (float)(e0 * W);
        pool[j][2][c] = t1 / (float)((H - s1) * W);
    }
    __syncthreads();
    const float* wb[3] = {wg, w0, w1};
    const float* bb[3] = {bg, b0, b1};
    float v[HEAD_CROPS][3];
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        float acc[HEAD_CROPS];
#pragma unroll
        for (int j = 0; j < HEAD_CROPS; ++j) acc[j] = 0.f;
        for (int k = 0; k < C; ++k) {
            const float wv = __ldg(wb[b] + (size_t)k * C + c);
#pragma unroll
            for (int j = 0; j < HEAD_CROPS; ++j) acc[j] = fmaf(pool[j][b][k], wv, acc[j]);
        }
        const float bias = bb[b][c];
#pragma unroll
        for (int j = 0; j < HEAD_CROPS; ++j) v[j][b] = acc[j] + bias;
    }
#pragma unroll
    for (int j = 0; j < HEAD_CROPS; ++j) {
        float s = (v[j][0] * v[j][0] + v[j][1] * v[j][1]) + v[j][2] * v[j][2];
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) red[j][warp] = s;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < HEAD_CROPS; ++j) {
        if (j >= nc) break;
        float s = 0.f;
        for (int k = 0; k < WARPS; ++k) s += red[j][k];
        const float inv = 1.f / sqrtf(s);
        float* dst = out + (size_t)crops[off + n0 + j].out_row * out_ld + 3 * c;
        float* rw = raw ? raw + (size_t)(n0 + j) * FEAT + 3 * c : nullptr;
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            dst[b] = v[j][b] * inv;
            if (rw) rw[b] = v[j][b];
        }
    }
}

}  // namespace csp
}  // namespace bmb
