// vit_tc.cuh -- the non-GEMM kernels of the CLIP-ReID ViT-B/16 image encoder (reid/backbones/clip/clip/model.py
// VisionTransformer + make_model.py build_transformer, eval mode).  The linear layers (patch embedding, in_proj,
// out_proj, c_fc, c_proj) run on rn::k_conv_tc as 1x1 convolutions over a [crops x tokens] x 1 map; what is here:
//
//   k_vit_patchify    staged crop [H][W][3] -> patch rows [P][768], k = (ky * 16 + kx) * 3 + ci, 16x16 patches at a
//                     given stride (16 for CLIP; 12 for the overlapping patches of vit_tiny)
//   k_vit_layernorm   one warp per 768-wide token row, float32, two-pass mean / variance (eps 1e-5); the EMBED form
//                     builds the token first: row 0 is the class embedding, row t the patch row t - 1, plus the
//                     positional table (which carries the class embedding in its row 0), then ln_pre
//   k_vit_attention   fused multi-head attention of one (crop, head, query block): K and V of the head in shared
//                     memory, scores, max-subtracted float32 softmax and P.V, written head-interleaved into
//                     [tokens][width].  q arrives pre-scaled by 1/8 (folded into in_proj at export).  Instances:
//                     <768, 288> (CLIP) and <192, 320> (the ViT-Nano / ViT-Tiny family, 3 heads, up to 311 tokens)
//   k_vit_head        token 0 only: ln_post (its affine folded into the two BatchNorm1d), the 768x512 projection,
//                     the concatenation [bottleneck | bottleneck_proj] and the L2 normalisation, into the caller's row
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bmb {
namespace vit {

constexpr int D = 768;          // ViT-B/16 width
constexpr int HEADS = 12;
constexpr int HD = 64;          // head dim
constexpr int PATCH = 16;
constexpr int PROJ = 512;       // image_encoder.proj output
constexpr int FEAT = D + PROJ;  // 1280: cat(bottleneck(x0), bottleneck_proj(x0 @ proj))
constexpr int MAX_T = 288;      // tokens an attention CTA holds per lane (9 x 32); 257 at 256x256
constexpr int ATT_QB = 32;      // queries per attention CTA
constexpr int ATT_THREADS = 256;
constexpr float LN_EPS = 1e-5f;

// staged crops [n][H][W][3] -> patch rows [n][gh gw][768], gh = (H - 16) / stride + 1 (likewise gw): the 16x16 window
// of patch (py, px) starts at (py stride, px stride); one thread per float4 of output (768 = 192 x 4)
__global__ void k_vit_patchify(const float* __restrict__ crop, int H, int W, int stride, const int* __restrict__ d_n,
                               int off, int cap, float* __restrict__ out) {
    int n_crops = *d_n - off;
    n_crops = n_crops < 0 ? 0 : (n_crops > cap ? cap : n_crops);
    const int gw = (W - PATCH) / stride + 1, P = ((H - PATCH) / stride + 1) * gw;
    const size_t total = (size_t)n_crops * P * (D / 4);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int q = (int)(i % (D / 4));
        const size_t row = i / (D / 4);
        const int n = (int)(row / P), p = (int)(row - (size_t)n * P);
        const int py = p / gw, px = p - py * gw;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int k = 4 * q + e, tap = k / 3, ci = k - 3 * tap, ky = tap / PATCH, kx = tap - ky * PATCH;
            v[e] = crop[(((size_t)n * H + py * stride + ky) * W + px * stride + kx) * 3 + ci];
        }
        reinterpret_cast<float4*>(out)[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// sum over a warp, the same butterfly order on every lane (every lane gets the identical total)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// out[r] = LN(x[r]) * gamma + beta over `rows_per_crop` token rows of every crop in the chunk.  EMBED: x[r] is built
// from the patch-embedding rows `in` ([crops][T - 1][768]) and the positional table `pos` ([T][768]).
template <bool EMBED>
__global__ void __launch_bounds__(256) k_vit_layernorm(const float* __restrict__ in, const float* __restrict__ pos,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       int T, const int* __restrict__ d_n, int off, int cap,
                                                       float* __restrict__ out) {
    int n_crops = *d_n - off;
    n_crops = n_crops < 0 ? 0 : (n_crops > cap ? cap : n_crops);
    const int lane = threadIdx.x & 31;
    const size_t rows = (size_t)n_crops * T;
    for (size_t r = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; r < rows;
         r += ((size_t)gridDim.x * blockDim.x) >> 5) {
        float4 v[6];
        if (EMBED) {
            const int n = (int)(r / T), t = (int)(r - (size_t)n * T);
            const float4* pr = reinterpret_cast<const float4*>(pos + (size_t)t * D);
            const float4* xr = reinterpret_cast<const float4*>(in + ((size_t)n * (T - 1) + t - 1) * D);
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                v[i] = pr[lane + 32 * i];
                if (t > 0) {
                    const float4 x = xr[lane + 32 * i];
                    v[i].x = x.x + v[i].x; v[i].y = x.y + v[i].y; v[i].z = x.z + v[i].z; v[i].w = x.w + v[i].w;
                }
            }
        } else {
            const float4* xr = reinterpret_cast<const float4*>(in + r * D);
#pragma unroll
            for (int i = 0; i < 6; ++i) v[i] = xr[lane + 32 * i];
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        const float mean = warp_sum(s) * (1.f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + b * b) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + LN_EPS);
        float4* o = reinterpret_cast<float4*>(out + r * D);
        const float4* g = reinterpret_cast<const float4*>(gamma);
        const float4* b = reinterpret_cast<const float4*>(beta);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const float4 gg = g[lane + 32 * i], bb = b[lane + 32 * i];
            o[lane + 32 * i] = make_float4((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y,
                                           (v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w);
        }
    }
}

constexpr int KPAD = HD + 1;   // K rows padded to 65 floats: lane j reading k[j][d] hits bank (j + d) % 32

// floats of the padded K block, rounded up to a multiple of 4 so that V behind it stays 16-byte aligned (float4 stores)
__host__ __device__ inline size_t k_block_floats(int T) { return ((size_t)T * KPAD + 3) & ~(size_t)3; }

inline size_t attention_smem_bytes(int T) {
    return sizeof(float) * (k_block_floats(T) + (size_t)T * HD + (ATT_THREADS / 32) * ((size_t)T + HD));
}

// qkv [crops][T][3 * DM] (q | k | v, head h at columns 64 h .. 64 h + 63 of each), out [crops][T][DM], T <= MAXT.
// grid (ceil(T / ATT_QB), DM / 64, crops); each warp walks its queries one at a time: lane j holds scores j, j + 32, ...
template <int DM, int MAXT>
__global__ void __launch_bounds__(ATT_THREADS) k_vit_attention(const float* __restrict__ qkv, int T,
                                                               const int* __restrict__ d_n, int off, int cap,
                                                               float* __restrict__ out) {
    int n_crops = *d_n - off;
    n_crops = n_crops < 0 ? 0 : (n_crops > cap ? cap : n_crops);
    const int n = blockIdx.z, h = blockIdx.y;
    if (n >= n_crops) return;
    extern __shared__ __align__(16) float sm[];
    float* sK = sm;                        // [T][65]
    float* sV = sK + k_block_floats(T);    // [T][64]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* sP = sV + (size_t)T * HD + (size_t)warp * (T + HD);   // this warp's probabilities [T] and query [64]
    float* sQ = sP + T;
    const float* base = qkv + (size_t)n * T * 3 * DM;
    for (int i = threadIdx.x; i < T * (HD / 4); i += blockDim.x) {
        const int t = i / (HD / 4), c = 4 * (i - t * (HD / 4));
        const float4 k = *reinterpret_cast<const float4*>(base + (size_t)t * 3 * DM + DM + h * HD + c);
        const float4 v = *reinterpret_cast<const float4*>(base + (size_t)t * 3 * DM + 2 * DM + h * HD + c);
        float* kr = sK + t * KPAD + c;
        kr[0] = k.x; kr[1] = k.y; kr[2] = k.z; kr[3] = k.w;
        *reinterpret_cast<float4*>(sV + t * HD + c) = v;
    }
    __syncthreads();
    constexpr int NJ = MAXT / 32;
    const int q_end = min(T, (int)(blockIdx.x + 1) * ATT_QB);
    for (int t = blockIdx.x * ATT_QB + warp; t < q_end; t += ATT_THREADS / 32) {
        const float* qr = base + (size_t)t * 3 * DM + h * HD;
        sQ[lane] = qr[lane];
        sQ[lane + 32] = qr[lane + 32];
        __syncwarp();
        float s[NJ];
#pragma unroll
        for (int u = 0; u < NJ; ++u) s[u] = -INFINITY;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
            const int j = lane + 32 * u;
            if (j < T) {
                const float* kr = sK + j * KPAD;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
                for (int d = 0; d < HD; d += 4) {
                    a0 = fmaf(sQ[d], kr[d], a0);
                    a1 = fmaf(sQ[d + 1], kr[d + 1], a1);
                    a2 = fmaf(sQ[d + 2], kr[d + 2], a2);
                    a3 = fmaf(sQ[d + 3], kr[d + 3], a3);
                }
                s[u] = (a0 + a1) + (a2 + a3);
            }
        }
        float mx = s[0];
#pragma unroll
        for (int u = 1; u < NJ; ++u) mx = fmaxf(mx, s[u]);
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int u = 0; u < NJ; ++u) {
            const int j = lane + 32 * u;
            if (j < T) {
                const float p = expf(s[u] - mx);
                sum += p;
                sP[j] = p;
            }
        }
        const float inv = 1.f / warp_sum(sum);
        __syncwarp();
        float o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f;
        int j = 0;
        for (; j + 1 < T; j += 2) {
            const float p0 = sP[j], p1 = sP[j + 1];
            o0 = fmaf(p0, sV[j * HD + lane], o0);
            o1 = fmaf(p0, sV[j * HD + lane + 32], o1);
            o2 = fmaf(p1, sV[(j + 1) * HD + lane], o2);
            o3 = fmaf(p1, sV[(j + 1) * HD + lane + 32], o3);
        }
        if (j < T) {
            o0 = fmaf(sP[j], sV[j * HD + lane], o0);
            o1 = fmaf(sP[j], sV[j * HD + lane + 32], o1);
        }
        float* orow = out + ((size_t)n * T + t) * DM + h * HD;
        orow[lane] = (o0 + o2) * inv;
        orow[lane + 32] = (o1 + o3) * inv;
        __syncwarp();   // sQ / sP are rewritten by this warp's next query
    }
}

// Head, one CTA (256 threads) per crop.  x: the residual stream after the last block ([crops][T][768], token 0 used).
// g768 / b768: ln_post's affine folded into bottleneck; wproj [768][512] K-major and bproj: ln_post's affine, proj and
// bottleneck_proj folded.  Writes the L2-normalised 1280-d row to out + crops[off + n].out_row * out_ld, or, when
// `tap` is set, the un-normalised row to tap + n * 1280.
__global__ void __launch_bounds__(256) k_vit_head(const float* __restrict__ x, int T, const float* __restrict__ g768,
                                                  const float* __restrict__ b768, const float* __restrict__ wproj,
                                                  const float* __restrict__ bproj, const CropDesc* __restrict__ crops,
                                                  const int* __restrict__ d_n, int off, int cap,
                                                  float* __restrict__ out, int out_ld, float* __restrict__ tap) {
    int n_crops = *d_n - off;
    n_crops = n_crops < 0 ? 0 : (n_crops > cap ? cap : n_crops);
    const int n = blockIdx.x;
    if (n >= n_crops) return;
    __shared__ __align__(16) float xh[D];
    __shared__ float f[FEAT];
    __shared__ float red[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0) {   // LayerNorm of token 0 without its affine
        const float4* xr = reinterpret_cast<const float4*>(x + (size_t)n * T * D);
        float4 v[6];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) { v[i] = xr[lane + 32 * i]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
        const float mean = warp_sum(s) * (1.f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + b * b) + (c * c + d * d);
        }
        const float rstd = rsqrtf(warp_sum(q) * (1.f / D) + LN_EPS);
#pragma unroll
        for (int i = 0; i < 6; ++i)
            reinterpret_cast<float4*>(xh)[lane + 32 * i] = make_float4((v[i].x - mean) * rstd, (v[i].y - mean) * rstd,
                                                                       (v[i].z - mean) * rstd, (v[i].w - mean) * rstd);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < D; c += blockDim.x) f[c] = fmaf(xh[c], g768[c], b768[c]);
    for (int c = threadIdx.x; c < PROJ; c += blockDim.x) {
        float t[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = 0; k < D; k += 4) {
#pragma unroll
            for (int u = 0; u < 4; ++u) t[u] = fmaf(xh[k + u], wproj[(size_t)(k + u) * PROJ + c], t[u]);
        }
        f[D + c] = bproj[c] + ((t[0] + t[1]) + (t[2] + t[3]));
    }
    __syncthreads();
    float sq = 0.f;
    for (int c = threadIdx.x; c < FEAT; c += blockDim.x) sq += f[c] * f[c];
    sq = warp_sum(sq);
    if (lane == 0) red[warp] = sq;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    if (tap) {
        for (int c = threadIdx.x; c < FEAT; c += blockDim.x) tap[(size_t)n * FEAT + c] = f[c];
        return;
    }
    const float nrm = sqrtf(tot);
    float* dst = out + (size_t)crops[off + n].out_row * out_ld;
    for (int c = threadIdx.x; c < FEAT; c += blockDim.x) dst[c] = f[c] / nrm;
}

}  // namespace vit
}  // namespace bmb
