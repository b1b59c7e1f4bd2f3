// lmbn_head.cuh -- the LMBN_n head (reid/backbones/lmbn/lmbn_n.py:96-146, eval mode): poolings of the three branch
// outputs, the seven BNNeck vectors, the interleaved 3584-d row and its L2 normalisation.  Included by reid_model.cu.
//
// pooled[crop][6][C] (C = 512):  0 average and 1 max of the bottleneck output (glo == glo_drop in eval),
//                                2 max, 3 average of the top half rows, 4 average of the bottom half of the partial
//                                branch, 5 average of the channel branch.
// Output vector k (0..6) is written interleaved: row[c * 7 + k] (torch.stack(..., dim=2).flatten(1, 2)).
#pragma once

namespace bmb {

constexpr int LMBN_C = 512, LMBN_VECS = 7, LMBN_POOLS = 6;

// K9: per crop, the poolings of one branch output x [crops][H][W][C] into its slots of `pooled`.
// which: 0 bottleneck (slots 0, 1), 1 partial branch (slots 2, 3, 4), 2 channel branch (slot 5).
// A thread owns a channel and walks the pixels in order: coalesced over channels, deterministic sums.
__global__ void __launch_bounds__(256) k_lmbn_pool(const float* __restrict__ x, int H, int W, int C, int which,
                                                   float* __restrict__ pooled, const int* __restrict__ d_n, int off,
                                                   int cap) {
    const int n = blockIdx.x;
    if (n >= chunk_count(d_n, off, cap)) return;
    const float* xp = x + (size_t)n * H * W * C;
    float* dst = pooled + (size_t)n * LMBN_POOLS * C;
    const int half = (H / 2) * W, HW = H * W;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float top = 0.f, bot = 0.f, mx = -INFINITY;
        for (int p = 0; p < half; ++p) {
            const float v = xp[(size_t)p * C + c];
            top += v;
            mx = fmaxf(mx, v);
        }
        for (int p = half; p < HW; ++p) {
            const float v = xp[(size_t)p * C + c];
            bot += v;
            mx = fmaxf(mx, v);
        }
        if (which == 0) {
            dst[c] = (top + bot) / (float)HW;
            dst[C + c] = mx;
        } else if (which == 1) {
            dst[2 * C + c] = mx;
            dst[3 * C + c] = top / (float)half;
            dst[4 * C + c] = bot / (float)(HW - half);
        } else {
            dst[5 * C + c] = (top + bot) / (float)HW;
        }
    }
}

struct NeckArgs {
    const float* w[5];   // reduction necks in output-vector order, 1x1 with BatchNorm1d folded: [C][C] K-major
    const float* b[5];   // [C]
    const float* wsh;    // shared: [C/2][C] with shared.1 folded
    const float* bsh;    // [C]
    const float* chst;   // reduction_ch_0 scale, shift, reduction_ch_1 scale, shift: [4][C]
};

constexpr int NECK_COLS = 32, NECK_ROWS = 8;
constexpr size_t NECK_SMEM = sizeof(float) * ((size_t)LMBN_C * NECK_COLS + (size_t)NECK_ROWS * LMBN_C);

// K10: the neck GEMMs of a whole chunk.  grid = (C / 32 column slices, 6 matrices): matrix k < 5 maps pooled slot k of
// every crop to output vector k; matrix 5 (`shared`) maps both 256-channel halves of every crop's channel-branch
// average (2 rows per crop) to vectors 5 and 6, with ReLU and the reduction_ch BatchNorm1d.  A CTA stages its
// [K][32] weight slice once and streams the crops through it, so every weight is read once per chunk.  Warp r of a
// pass computes row r0 + r, lane j output column j (input row broadcast, weight row conflict-free).
__global__ void __launch_bounds__(256) k_lmbn_neck(const NeckArgs a, const float* __restrict__ pooled,
                                                   const CropDesc* __restrict__ crops, const int* __restrict__ d_n,
                                                   int off, int cap, float* __restrict__ out, int out_ld) {
    constexpr int C = LMBN_C;
    const int mat = blockIdx.y, c0 = blockIdx.x * NECK_COLS;
    const int K = mat < 5 ? C : C / 2;
    extern __shared__ __align__(16) float smem[];
    float* sw = smem;                           // [K][32]
    float* sx = smem + (size_t)C * NECK_COLS;   // [8][K]
    const float* w = a.wsh;
    const float* bias = a.bsh;
#pragma unroll
    for (int k = 0; k < 5; ++k)   // static indices keep the parameter arrays out of local memory
        if (k == mat) { w = a.w[k]; bias = a.b[k]; }
    for (int e = threadIdx.x; e < K * NECK_COLS; e += blockDim.x) {
        const int k = e / NECK_COLS, j = e - k * NECK_COLS;
        sw[e] = w[(size_t)k * C + c0 + j];
    }
    const int n_crops = chunk_count(d_n, off, cap);
    const int rows = mat < 5 ? n_crops : 2 * n_crops;
    const int j = threadIdx.x & 31, r = threadIdx.x >> 5;
    const int c = c0 + j;
    for (int r0 = 0; r0 < rows; r0 += NECK_ROWS) {
        __syncthreads();
        for (int e = threadIdx.x; e < NECK_ROWS * K; e += blockDim.x) {
            const int rr = e / K, k = e - rr * K, row = r0 + rr;
            float v = 0.f;
            if (row < rows) {
                const int crop = mat < 5 ? row : row >> 1;
                const float* src = pooled + (size_t)crop * LMBN_POOLS * C + (mat < 5 ? mat * C : 5 * C + (row & 1) * (C / 2));
                v = src[k];
            }
            sx[e] = v;
        }
        __syncthreads();
        const int row = r0 + r;
        if (row >= rows) continue;
        const float* xr = sx + (size_t)r * K;
        float t0 = 0.f, t1 = 0.f, t2 = 0.f, t3 = 0.f;   // four independent chains, fixed combination order
        for (int k = 0; k < K; k += 4) {
            t0 = fmaf(xr[k], sw[k * NECK_COLS + j], t0);
            t1 = fmaf(xr[k + 1], sw[(k + 1) * NECK_COLS + j], t1);
            t2 = fmaf(xr[k + 2], sw[(k + 2) * NECK_COLS + j], t2);
            t3 = fmaf(xr[k + 3], sw[(k + 3) * NECK_COLS + j], t3);
        }
        const float acc = (t0 + t1) + (t2 + t3);
        float v;
        int vec, crop;
        if (mat < 5) {
            v = acc + bias[c];
            vec = mat;
            crop = row;
        } else {
            const int h = row & 1;
            v = fmaf(fmaxf(acc + bias[c], 0.f), a.chst[(2 * h) * C + c], a.chst[(2 * h + 1) * C + c]);
            vec = 5 + h;
            crop = row >> 1;
        }
        out[(size_t)crops[off + crop].out_row * out_ld + (size_t)c * LMBN_VECS + vec] = v;
    }
}

// K11: row-wise L2 normalisation of the finished rows in place (base_backend.py:197-207).  One CTA per crop.
__global__ void __launch_bounds__(256) k_l2_normalise(const CropDesc* __restrict__ crops, const int* __restrict__ d_n,
                                                      int off, int cap, float* __restrict__ out, int out_ld, int feat) {
    const int n = blockIdx.x;
    if (n >= chunk_count(d_n, off, cap)) return;
    __shared__ float red[32];
    float* dst = out + (size_t)crops[off + n].out_row * out_ld;
    float sq = 0.f;
    for (int f = threadIdx.x; f < feat; f += blockDim.x) sq = fmaf(dst[f], dst[f], sq);
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    const float nrm = sqrtf(tot);
    for (int f = threadIdx.x; f < feat; f += blockDim.x) dst[f] = dst[f] / nrm;
}

}  // namespace bmb
