// hacnn_kernels.cuh -- the float32 CUDA-core kernels of the HACNN ReID path (reid/backbones/hacnn.py, eval mode).
// Every ConvBlock after the stem runs on rn::k_conv_tc; these kernels do the rest.  All maps are NHWC; the local
// branch keeps its four regions as one batch laid out [crop][region].
//   k_stem        the 3 -> 32 3x3 stride-2 ConvBlock (BN and bias folded, ReLU) on the 160x64 crop.
//   k_pool3       3x3 pad-1 pools with PyTorch's output size (H - 1) / stride + 1: the average at stride 1
//                 (count_include_pad, so always / 9) and the max at stride 2 (odd maps too: 6x7 -> 3x4).
//   k_attn        per crop: the channel mean of every pixel and the average pool of every channel, then the spatial
//                 3x3 stride-2 ConvBlock, the x2 align_corners resize and the scalar ConvBlock into s[p]; the channel
//                 MLP, v = W c with W the soft attention's folded 1x1; and theta = tanh(fc(pool)).
//   k_attn_apply  x[p][o] *= sigmoid(relu(s[p] v[o] + b[o])): the soft attention's 1x1 ConvBlock over the rank-1
//                 map s (x) c is s[p] (W c)[o] + b[o], which spares a C x C GEMM over every pixel.
//   k_stn         the four regions' affine_grid + grid_sample (align_corners=False, zero padding) of the previous
//                 level's map, resized (align_corners=True) to the local map's size and added to the previous local
//                 map: each output pixel takes the bilinear taps of the four STN samples around it, so the full-size
//                 STN map never exists.
//   k_head_pool   the two heads' average pools; k_head the two half-row L2 norms, the final norm and the scatter.
// Reductions run in a fixed order without atomics, so a crop's row never depends on its place in a chunk.
#pragma once
#include <cuda_runtime.h>

#include "mlfn_kernels.cuh"

namespace bmb {
namespace hacnn {

using mlfn::crops_in_chunk;

constexpr int IN_H = 160, IN_W = 64;
constexpr int STEM_C = 32;
constexpr int FEAT = 1024;
constexpr int HALF = 512;
constexpr int C3 = 384;
constexpr int MAX_HW = 40 * 16;   // the largest attended map (inception1's output)
constexpr int MAX_C = 384;
constexpr int THETA = 24;         // per crop: 3 levels x 4 regions x (tx, ty)

// The soft / hard attention parameters of one level in d_w (fold_hacnn's order): sp = [9 taps, bias, scale, shift]
struct AttnW {
    const float *sp, *w1, *b1, *w2, *b2, *wv, *bv, *wfc, *bfc;
};

__global__ void k_count4(const int* __restrict__ d_n, int* __restrict__ d_n4) { *d_n4 = 4 * *d_n; }

// blob [crops][160][64][3] -> out [crops][80][32][32]; w [27][32] (k = (kh*3 + kw)*3 + ci), b [32]; one thread per
// output pixel and channel quad
__global__ void __launch_bounds__(256) k_stem(const float* __restrict__ blob, const float* __restrict__ w,
                                              const float* __restrict__ b, const int* __restrict__ d_n, int off, int cap,
                                              float* __restrict__ out) {
    constexpr int HO = IN_H / 2, WO = IN_W / 2, CQ = STEM_C / 4;
    const size_t items = (size_t)crops_in_chunk(d_n, off, cap) * HO * WO * CQ;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(it % CQ);
        const size_t px = it / CQ;
        const int ox = (int)(px % WO), oy = (int)(px / WO % HO), n = (int)(px / (WO * HO));
        const float* src = blob + (size_t)n * IN_H * IN_W * 3;
        float4 acc = __ldg(reinterpret_cast<const float4*>(b) + q);
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = 2 * oy + ky - 1;
            if (iy < 0 || iy >= IN_H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = 2 * ox + kx - 1;
                if (ix < 0 || ix >= IN_W) continue;
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) {
                    const float a = src[((size_t)iy * IN_W + ix) * 3 + ci];
                    const float4 wv = __ldg(reinterpret_cast<const float4*>(w + ((ky * 3 + kx) * 3 + ci) * STEM_C) + q);
                    acc.x = fmaf(a, wv.x, acc.x); acc.y = fmaf(a, wv.y, acc.y);
                    acc.z = fmaf(a, wv.z, acc.z); acc.w = fmaf(a, wv.w, acc.w);
                }
            }
        }
        acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
        reinterpret_cast<float4*>(out)[it] = acc;
    }
}

// in [imgs][H][W][C] -> out [imgs][Ho][Wo][C], 3x3 pad 1, Ho = (H - 1) / stride + 1; MAX: max over the taps inside the
// map, else the sum of the taps inside the map / 9 (count_include_pad).  C a multiple of 4.
template <bool MAX>
__global__ void __launch_bounds__(256) k_pool3(const float* __restrict__ in, int H, int W, int C, int stride,
                                               const int* __restrict__ d_n, int off, int cap, float* __restrict__ out) {
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1, cq = C / 4;
    const size_t items = (size_t)crops_in_chunk(d_n, off, cap) * Ho * Wo * cq;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(it % cq);
        const size_t px = it / cq;
        const int ox = (int)(px % Wo), oy = (int)(px / Wo % Ho), n = (int)(px / ((size_t)Wo * Ho));
        const float* src = in + (size_t)n * H * W * C + 4 * q;
        float4 r = MAX ? make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY) : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * stride + ky - 1;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * stride + kx - 1;
                if (ix < 0 || ix >= W) continue;
                const float4 v = __ldg(reinterpret_cast<const float4*>(src + ((size_t)iy * W + ix) * C));
                if (MAX) {
                    r.x = fmaxf(r.x, v.x); r.y = fmaxf(r.y, v.y); r.z = fmaxf(r.z, v.z); r.w = fmaxf(r.w, v.w);
                } else {
                    r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w;
                }
            }
        }
        if (!MAX) { r.x /= 9.f; r.y /= 9.f; r.z /= 9.f; r.w /= 9.f; }
        reinterpret_cast<float4*>(out)[it] = r;
    }
}

// x [crops][H][W][C] (H, W even, H W <= MAX_HW, C <= MAX_C, C % 16 == 0) -> s [crops][H W], v [crops][C],
// theta[n * THETA + 8 level + k].  One CTA of 256 threads per crop.
__global__ void __launch_bounds__(256) k_attn(const float* __restrict__ x, int H, int W, int C, const AttnW a,
                                              int level, const int* __restrict__ d_n, int off, int cap,
                                              float* __restrict__ s_out, float* __restrict__ v_out,
                                              float* __restrict__ theta) {
    const int n = blockIdx.x;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    __shared__ float sm[MAX_HW], sq[MAX_HW / 4], sg[MAX_C], sh[MAX_C / 16], sc[MAX_C];
    const int HW = H * W, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, Hq = H / 2, Wq = W / 2, R = C / 16;
    const float* xs = x + (size_t)n * HW * C;
    for (int p = warp; p < HW; p += 8) {   // channel mean of pixel p: one warp, lanes over channel quads
        float t = 0.f;
        for (int q = lane; q < C / 4; q += 32) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(xs + (size_t)p * C) + q);
            t += (v.x + v.y) + (v.z + v.w);
        }
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) sm[p] = t / (float)C;
    }
    for (int c = tid; c < C; c += 256) {   // average pool of channel c
        float t = 0.f;
        for (int p = 0; p < HW; ++p) t += xs[(size_t)p * C + c];
        sg[c] = t / (float)HW;
    }
    __syncthreads();
    for (int i = tid; i < Hq * Wq; i += 256) {   // spatial 3x3 stride-2 ConvBlock (1 -> 1) + ReLU
        const int oy = i / Wq, ox = i - oy * Wq;
        float t = a.sp[9];
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx) {
                const int iy = 2 * oy + ky - 1, ix = 2 * ox + kx - 1;
                if (iy >= 0 && iy < H && ix >= 0 && ix < W) t = fmaf(a.sp[ky * 3 + kx], sm[iy * W + ix], t);
            }
        sq[i] = fmaxf(t, 0.f);
    }
    for (int j = tid; j < R; j += 256) {   // channel attention, first ConvBlock (C -> C / 16)
        float t = a.b1[j];
        for (int c = 0; c < C; ++c) t = fmaf(sg[c], a.w1[(size_t)c * R + j], t);
        sh[j] = fmaxf(t, 0.f);
    }
    if (tid < 8) {   // hard attention: theta = tanh(fc(pool))
        float t = a.bfc[tid];
        for (int c = 0; c < C; ++c) t = fmaf(sg[c], a.wfc[c * 8 + tid], t);
        theta[(size_t)n * THETA + 8 * level + tid] = tanhf(t);
    }
    __syncthreads();
    const float fy = (float)(Hq - 1) / (float)(H - 1), fx = (float)(Wq - 1) / (float)(W - 1);
    for (int p = tid; p < HW; p += 256) {   // x2 bilinear resize (align_corners=True), then the scalar ConvBlock
        const int y = p / W, xx = p - y * W;
        const float sy = fy * y, sx = fx * xx;
        const int y0 = (int)sy, x0 = (int)sx;
        const int y1 = y0 + (y0 < Hq - 1), x1 = x0 + (x0 < Wq - 1);
        const float ly = sy - y0, lx = sx - x0;
        const float up = (1.f - ly) * ((1.f - lx) * sq[y0 * Wq + x0] + lx * sq[y0 * Wq + x1]) +
                         ly * ((1.f - lx) * sq[y1 * Wq + x0] + lx * sq[y1 * Wq + x1]);
        s_out[(size_t)n * HW + p] = fmaxf(fmaf(a.sp[10], up, a.sp[11]), 0.f);
    }
    for (int o = tid; o < C; o += 256) {   // channel attention, second ConvBlock (C / 16 -> C)
        float t = a.b2[o];
        for (int j = 0; j < R; ++j) t = fmaf(sh[j], a.w2[(size_t)j * C + o], t);
        sc[o] = fmaxf(t, 0.f);
    }
    __syncthreads();
    for (int o = tid; o < C; o += 256) {   // v = W c with W the soft attention's folded 1x1 (K-major [C][C])
        float t0 = 0.f, t1 = 0.f;
        for (int i = 0; i < C; i += 2) {
            t0 = fmaf(sc[i], a.wv[(size_t)i * C + o], t0);
            t1 = fmaf(sc[i + 1], a.wv[(size_t)(i + 1) * C + o], t1);
        }
        v_out[(size_t)n * C + o] = t0 + t1;
    }
}

// x [crops][HW][C] *= sigmoid(relu(s[p] v[o] + b[o])), in place
__global__ void __launch_bounds__(256) k_attn_apply(float* __restrict__ x, int HW, int C, const float* __restrict__ s,
                                                    const float* __restrict__ v, const float* __restrict__ b,
                                                    const int* __restrict__ d_n, int off, int cap) {
    const int cq = C / 4;
    const size_t items = (size_t)crops_in_chunk(d_n, off, cap) * HW * cq;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(it % cq);
        const size_t px = it / cq;
        const int n = (int)(px / HW);
        const float sp = s[px];
        const float4 vv = __ldg(reinterpret_cast<const float4*>(v + (size_t)n * C) + q);
        const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + q);
        float4 o = reinterpret_cast<float4*>(x)[it];
        o.x *= 1.f / (1.f + expf(-fmaxf(fmaf(sp, vv.x, bb.x), 0.f)));
        o.y *= 1.f / (1.f + expf(-fmaxf(fmaf(sp, vv.y, bb.y), 0.f)));
        o.z *= 1.f / (1.f + expf(-fmaxf(fmaf(sp, vv.z, bb.z), 0.f)));
        o.w *= 1.f / (1.f + expf(-fmaxf(fmaf(sp, vv.w, bb.w), 0.f)));
        reinterpret_cast<float4*>(x)[it] = o;
    }
}

// acc += wgt * (bilinear sample of src [H][W][C] at (iy, ix), channel quad q), zero outside the map (grid_sample's
// zero padding)
__device__ __forceinline__ void add_sample(float4& acc, float wgt, const float* __restrict__ src, int H, int W, int C,
                                           int q, float iy, float ix) {
    const float y0f = floorf(iy), x0f = floorf(ix);
    const int y0 = (int)y0f, x0 = (int)x0f;
    const float ly = iy - y0f, lx = ix - x0f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int yy = y0 + (t >> 1), xx = x0 + (t & 1);
        if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
        const float w = wgt * ((t >> 1) ? ly : 1.f - ly) * ((t & 1) ? lx : 1.f - lx);
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + ((size_t)yy * W + xx) * C) + q);
        acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
    }
}

// src [crops][H][W][C], theta row n at theta + n * THETA (region r: tx = [2r], ty = [2r + 1]) -> out
// [crops][4][h][w][C] = resize_align_corners(STN_r(src), h x w) (+ prev [crops][4][h][w][C] when non-null).
// STN_r(src)[k][j] samples src at ix = j + tx W / 2, iy = ((0.25 y_k + ty + 1) H - 1) / 2, y_k = (2k + 1) / H - 1.
__global__ void __launch_bounds__(256) k_stn(const float* __restrict__ src, int H, int W, int C,
                                             const float* __restrict__ theta, const float* __restrict__ prev, int h,
                                             int w, const int* __restrict__ d_n, int off, int cap,
                                             float* __restrict__ out) {
    const int cq = C / 4;
    const int items = crops_in_chunk(d_n, off, cap) * 4 * h * w * cq;   // < 2^31: at most 1024 crops of 4 x 24x28x64
    const float fy = (float)(H - 1) / (float)(h - 1), fx = (float)(W - 1) / (float)(w - 1);
    for (int it = blockIdx.x * blockDim.x + threadIdx.x; it < items; it += gridDim.x * blockDim.x) {
        const int q = it % cq, px = it / cq;
        const int x = px % w, y = px / w % h, nr = px / (w * h);
        const int n = nr >> 2, r = nr & 3;
        const float tx = theta[(size_t)n * THETA + 2 * r], ty = theta[(size_t)n * THETA + 2 * r + 1];
        const float sy = fy * y, sx = fx * x;
        const int k0 = (int)sy, j0 = (int)sx;
        const int k1 = k0 + (k0 < H - 1), j1 = j0 + (j0 < W - 1);
        const float ly = sy - k0, lx = sx - j0;
        const float* s = src + (size_t)n * H * W * C;
        const float sxt = tx * (float)W * 0.5f;
        const float iy0 = ((0.25f * ((2 * k0 + 1) / (float)H - 1.f) + ty + 1.f) * H - 1.f) * 0.5f;
        const float iy1 = ((0.25f * ((2 * k1 + 1) / (float)H - 1.f) + ty + 1.f) * H - 1.f) * 0.5f;
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        add_sample(o, (1.f - ly) * (1.f - lx), s, H, W, C, q, iy0, j0 + sxt);
        add_sample(o, (1.f - ly) * lx, s, H, W, C, q, iy0, j1 + sxt);
        add_sample(o, ly * (1.f - lx), s, H, W, C, q, iy1, j0 + sxt);
        add_sample(o, ly * lx, s, H, W, C, q, iy1, j1 + sxt);
        if (prev) {
            const float4 p = reinterpret_cast<const float4*>(prev)[it];
            o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
        }
        reinterpret_cast<float4*>(out)[it] = o;
    }
}

// x3 [crops][HW3][384] -> pg [crops][384]; loc [crops][4][HWl][384] -> pl [crops][4 x 384] (region-major, the order
// of fc_local's input).  One CTA per crop.
__global__ void __launch_bounds__(256) k_head_pool(const float* __restrict__ x3, int HW3, const float* __restrict__ loc,
                                                   int HWl, const int* __restrict__ d_n, int off, int cap,
                                                   float* __restrict__ pg, float* __restrict__ pl) {
    const int n = blockIdx.x;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    for (int c = threadIdx.x; c < C3; c += 256) {
        const float* s = x3 + (size_t)n * HW3 * C3 + c;
        float t = 0.f;
        for (int p = 0; p < HW3; ++p) t += s[(size_t)p * C3];
        pg[(size_t)n * C3 + c] = t / (float)HW3;
    }
    for (int i = threadIdx.x; i < 4 * C3; i += 256) {
        const int r = i / C3, c = i - r * C3;
        const float* s = loc + ((size_t)(4 * n + r) * HWl) * C3 + c;
        float t = 0.f;
        for (int p = 0; p < HWl; ++p) t += s[(size_t)p * C3];
        pl[(size_t)n * 4 * C3 + i] = t / (float)HWl;
    }
}

__device__ __forceinline__ float block_sum(float v, float* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    return t;
}

// v [crops][1024] = [fc_global | fc_local] -> e = [g / |g|, l / |l|] / |[g / |g|, l / |l|]| into row
// crops[off + n].out_row.  One CTA of 256 threads per crop: elements t, t + 256 of each half.
template <typename Crop>
__global__ void __launch_bounds__(256) k_head(const float* __restrict__ v, const Crop* __restrict__ crops,
                                              const int* __restrict__ d_n, int off, int cap, float* __restrict__ out,
                                              int out_ld) {
    const int n = blockIdx.x;
    if (n >= crops_in_chunk(d_n, off, cap)) return;
    __shared__ float red[8];
    const float* src = v + (size_t)n * FEAT;
    float e[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) e[k] = src[threadIdx.x + 256 * k];
    const float ng = sqrtf(block_sum(e[0] * e[0] + e[1] * e[1], red));
    const float nl = sqrtf(block_sum(e[2] * e[2] + e[3] * e[3], red));
    e[0] /= ng; e[1] /= ng; e[2] /= nl; e[3] /= nl;
    const float nt = sqrtf(block_sum((e[0] * e[0] + e[1] * e[1]) + (e[2] * e[2] + e[3] * e[3]), red));
    float* dst = out + (size_t)crops[off + n].out_row * out_ld;
#pragma unroll
    for (int k = 0; k < 4; ++k) dst[threadIdx.x + 256 * k] = e[k] / nt;
}

}  // namespace hacnn
}  // namespace bmb
