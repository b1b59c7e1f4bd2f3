// resnet_tc.cuh -- every convolution of a ResNet Bottleneck after the stem as one implicit GEMM on the Hopper tensor
// cores (wgmma kind tf32, three-term split as in pointwise_tc.cuh, so the result keeps float32 accuracy):
//
//     a = a_hi + a_lo,  w = w_hi + w_lo   (hi = top 19 bits, lo = exact remainder)
//     D += A_hi*W_hi + A_hi*W_lo + A_lo*W_hi          (the dropped A_lo*W_lo term is ~2^-22 relative)
//
// GEMM view: M = output pixels x crops (flattened, so a tile may straddle crops), N = output channels, K = the taps of
// the main operand walked tap by tap (k = tap * C0 + ci) followed, for the fused conv3 + downsample, by the C1 channels
// of the strided 1x1 second operand.  Shapes covered: 1x1 stride 1 / 2, 3x3 stride 1 / 2 pad 1 (zero-filled borders),
// and [1x1 | strided 1x1] over the concatenated K.
//
// One CTA = 256 threads (two warpgroups) computes a BM = 128 x BN tile; warpgroup g owns rows 64 g .. 64 g + 63.  K is
// consumed in chunks of KC = 32 through a three-stage shared-memory ring:
//   * A: each thread cp.async-copies four 16-byte pieces (4 channels of one row) straight into the canonical no-swizzle
//     K-major layout (zero-fill for border taps and rows past M), then splits them in place into hi and a lo copy;
//   * B: the weights are packed at load time as [N / BN][K / KC][hi | lo][BN x KC canonical], so one bulk copy
//     (cp.async.bulk, completing on the stage's mbarrier) brings a chunk's hi and lo halves;
//   * chunk k + 1 is in flight while the MMAs of chunk k (and the tail of chunk k - 1) run; every wgmma is issued
//     unconditionally, with BN a template parameter.
// Epilogue: bias, optional residual, then relu = 0 none / 1 ReLU / 2 QuickGELU, float2 stores into NHWC [M][N].  The
// RELU_RES instances (relu = 3) compute relu(residual + relu(acc + bias)) instead: MLFN's fm_conv3, whose ReLU comes
// before the residual add.  They are separate instances so that the default ones keep their code.  The SLICE
// instances (HACNN's Inception streams, BN 32 / 64 / 128) store row m at out + m * out_ld instead of out + m * N, so
// that each stream writes its channel slice of the concatenated map in place (the caller offsets `out` by the slice's
// first channel).  The GELU instances (relu = 4, BN 64 / 128) apply the exact erf GELU of the ViT-Nano / ViT-Tiny MLP,
// x * 0.5 * (1 + erf(x / sqrt(2))), likewise separate so that no other instance's code changes.  The SILU instances
// (CSPReID-n's ConvBNSiLU, BN 32 / 64 / 128) apply x * sigmoid(x) after the bias (SILU = 1), or residual + silu(.) with
// the residual added after the activation (SILU = 2, a C3k2 bottleneck's shortcut).  They read the main operand, the
// residual and the output with the pixel pitches in_ld, res_ld and out_ld, so that a bottleneck reads and writes its
// channel slice of the C3k2 concatenation in place (the caller offsets each pointer by the slice's first channel).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>

#include "wgmma.cuh"

namespace bmb {
namespace rn {

constexpr int BM = 128;
constexpr int KC = 32;
constexpr int STAGES = 3;
constexpr int THREADS = 256;

struct ConvArgs {
    const float* in0;        // main operand, NHWC [crops][H0][W0][C0]
    const float* in1;        // second 1x1 operand (fused downsample), NHWC [crops][H1][W1][C1]; null when C1 == 0
    const float* w;          // packed weights (pack_conv_weights)
    const float* bias;       // [N]
    const float* residual;   // [M][N] or null
    float* out;              // [M][N]
    int H0, W0, C0, k0, s0;  // k0 in {1, 3} (pad k0 / 2), stride s0
    int H1, W1, C1, s1;
    int Ho, Wo, N, relu;     // relu: 0 none, 1 ReLU, 2 QuickGELU, 3 relu(residual + relu(.)) (RELU_RES instances),
                             // 4 exact GELU (GELU instances)
    int out_ld;              // SLICE / SILU instances: floats between output rows (0: the default [M][N] store)
    int in_ld, res_ld;       // SILU instances: floats between the pixels of in0 and between the rows of residual
};

// canonical (no swizzle, K-major) offset in floats of element (row, k) in a block whose K extent is KC
__device__ __host__ __forceinline__ int canon(int row, int k) { return (row >> 3) * (KC * 8) + (k >> 2) * 32 + (row & 7) * 4 + (k & 3); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

template <int BN>
constexpr size_t smem_bytes() {
    return sizeof(float) * (size_t)STAGES * (2 * BM * KC + 2 * BN * KC) + 128;
}

template <int BN, bool RELU_RES = false, bool SLICE = false, bool GELU = false, int SILU = 0>
__global__ void __launch_bounds__(THREADS, 1) k_conv_tc(const ConvArgs a, const int* __restrict__ d_n, int off, int cap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar[STAGES];
    int n_crops = *d_n - off;
    n_crops = n_crops < 0 ? 0 : (n_crops > cap ? cap : n_crops);
    const int HWo = a.Ho * a.Wo;
    const int M = n_crops * HWo;
    const int m0 = blockIdx.x * BM;
    if (m0 >= M) return;
    const int n0 = blockIdx.y * BN;
    const int K0 = a.k0 * a.k0 * a.C0, K = K0 + a.C1, nk = K / KC;
    const int pad = a.k0 >> 1;

    float* sA = reinterpret_cast<float*>(smem_raw);          // [STAGES][hi | lo][BM x KC]
    float* sB = sA + (size_t)STAGES * 2 * BM * KC;            // [STAGES][hi | lo][BN x KC]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;

    // the four rows this thread stages (row tid / 8 + 32 i, channels 4 (tid % 8) .. + 3 of every chunk)
    int rn_[4], ry[4], rx[4];
    bool rv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + (tid >> 3) + 32 * i;
        rv[i] = m < M;
        const int mm = rv[i] ? m : 0;
        rn_[i] = mm / HWo;
        const int p = mm - rn_[i] * HWo;
        ry[i] = p / a.Wo;
        rx[i] = p - ry[i] * a.Wo;
    }
    const int kq = (tid & 7) * 4;

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) um::mbar_init(&bar[s], 1);
        um::fence_mbar_init();
    }
    __syncthreads();

    const uint32_t bbytes = (uint32_t)(2 * BN * KC * sizeof(float));
    const float* wtile = a.w + (size_t)blockIdx.y * nk * 2 * BN * KC;
    auto issue = [&](int kk) {
        const int s = kk % STAGES;
        float* dst = sA + (size_t)s * 2 * BM * KC;
        const int k = kk * KC + kq;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float* src = a.in0;
            bool ok = rv[i];
            if (k < K0) {
                const int tap = k / a.C0, ci = k - tap * a.C0;
                const int ky = tap / a.k0, kx = tap - ky * a.k0;
                const int iy = ry[i] * a.s0 + ky - pad, ix = rx[i] * a.s0 + kx - pad;
                ok = ok && iy >= 0 && iy < a.H0 && ix >= 0 && ix < a.W0;
                if (ok) src = a.in0 + (((size_t)rn_[i] * a.H0 + iy) * a.W0 + ix) * (SILU ? a.in_ld : a.C0) + ci;
            } else {
                const int ci = k - K0;
                if (ok) src = a.in1 + (((size_t)rn_[i] * a.H1 + ry[i] * a.s1) * a.W1 + rx[i] * a.s1) * a.C1 + ci;
            }
            cp_async16(um::smem_u32(dst + canon((tid >> 3) + 32 * i, kq)), src, ok ? 16u : 0u);
        }
        cp_async_commit();
        if (tid == 0) {
            um::mbar_expect_tx(&bar[s], bbytes);
            um::bulk_g2s(sB + (size_t)s * 2 * BN * KC, wtile + (size_t)kk * 2 * BN * KC, bbytes, &bar[s]);
        }
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

    issue(0);
    constexpr uint32_t SBO_A = KC * 32, SBO_B = KC * 32;   // bytes between 8-row groups
    for (int kk = 0; kk < nk; ++kk) {
        const int s = kk % STAGES;
        float* hi = sA + (size_t)s * 2 * BM * KC;
        float* lo = hi + BM * KC;
        cp_async_wait_all();
#pragma unroll
        for (int i = 0; i < 4; ++i) {   // split this thread's own pieces: hi in place, lo beside it
            const int o = canon((tid >> 3) + 32 * i, kq);
            const float4 v = *reinterpret_cast<const float4*>(hi + o);
            float4 h, l;
            h.x = __uint_as_float(__float_as_uint(v.x) & 0xffffe000u); l.x = v.x - h.x;
            h.y = __uint_as_float(__float_as_uint(v.y) & 0xffffe000u); l.y = v.y - h.y;
            h.z = __uint_as_float(__float_as_uint(v.z) & 0xffffe000u); l.z = v.z - h.z;
            h.w = __uint_as_float(__float_as_uint(v.w) & 0xffffe000u); l.w = v.w - h.w;
            *reinterpret_cast<float4*>(hi + o) = h;
            *reinterpret_cast<float4*>(lo + o) = l;
        }
        um::fence_async_smem();
        um::mbar_wait(&bar[s], (uint32_t)(kk / STAGES) & 1u);
        // every thread's pieces of chunk kk are split, and both warpgroups have retired the MMAs of chunk kk - 2, whose
        // stage the loads of chunk kk + 1 overwrite
        __syncthreads();
        if (kk + 1 < nk) issue(kk + 1);
        const uint32_t a_hi = um::smem_u32(hi) + (uint32_t)wg * 8u * SBO_A, a_lo = um::smem_u32(lo) + (uint32_t)wg * 8u * SBO_A;
        const uint32_t b_hi = um::smem_u32(sB + (size_t)s * 2 * BN * KC), b_lo = b_hi + BN * KC * 4;
        um::wg_fence();
#pragma unroll
        for (int ks = 0; ks < KC; ks += 8) {
            const uint32_t o = (uint32_t)(ks >> 2) * 128;
            const uint64_t dah = um::make_desc(a_hi + o, 128, SBO_A), dal = um::make_desc(a_lo + o, 128, SBO_A);
            um::mma<BN, true>(acc, dah, b_hi + o, 128, SBO_B, 1u);
            um::mma<BN, true>(acc, dah, b_lo + o, 128, SBO_B, 1u);
            um::mma<BN, true>(acc, dal, b_hi + o, 128, SBO_B, 1u);
        }
        um::wg_commit();
        um::wg_wait<1>();
    }
    um::wg_wait<0>();
    um::wg_fence_acc<BN / 2>(acc);

    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + row + 8 * h;
        if (m >= M) continue;
        float* dst = a.out + (size_t)m * (SLICE || SILU ? a.out_ld : a.N) + n0;
        const float* res = a.residual ? a.residual + (size_t)m * (SILU ? a.res_ld : a.N) + n0 : nullptr;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            const int c = 8 * i + cq;
            const float2 b = *reinterpret_cast<const float2*>(a.bias + n0 + c);
            float2 o = make_float2(acc[4 * i + 2 * h] + b.x, acc[4 * i + 2 * h + 1] + b.y);
            if constexpr (SILU != 0) {
                o.x = o.x / (1.f + expf(-o.x)); o.y = o.y / (1.f + expf(-o.y));
                if constexpr (SILU == 2) {
                    const float2 r = *reinterpret_cast<const float2*>(res + c);
                    o.x += r.x; o.y += r.y;
                }
                *reinterpret_cast<float2*>(dst + c) = o;
                continue;
            }
            if constexpr (RELU_RES) {
                const float2 r = *reinterpret_cast<const float2*>(res + c);
                o.x = fmaxf(r.x + fmaxf(o.x, 0.f), 0.f); o.y = fmaxf(r.y + fmaxf(o.y, 0.f), 0.f);
                *reinterpret_cast<float2*>(dst + c) = o;
                continue;
            }
            if (res) {
                const float2 r = *reinterpret_cast<const float2*>(res + c);
                o.x += r.x; o.y += r.y;
            }
            if constexpr (GELU) {
                o.x = 0.5f * o.x * (1.f + erff(o.x * 0.70710678118654752f));
                o.y = 0.5f * o.y * (1.f + erff(o.y * 0.70710678118654752f));
            } else if (a.relu == 1) {
                o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f);
            } else if (a.relu == 2) {   // QuickGELU x * sigmoid(1.702 x) (CLIP's MLP)
                o.x = o.x / (1.f + expf(-1.702f * o.x)); o.y = o.y / (1.f + expf(-1.702f * o.y));
            }
            *reinterpret_cast<float2*>(dst + c) = o;
        }
    }
}

// output-channel tile of a layer: 128 when it divides N, else 64 (ResNet's layer1 conv1 / conv2), else 32 (HACNN's
// 32- and 96-wide streams and CSPReID-n's 32- and 96-wide bottleneck convs, SLICE and SILU instances only)
inline int tile_n(int N) { return N % 128 == 0 ? 128 : (N % 64 == 0 ? 64 : 32); }

// host: W [K][N] (K-major rows of N) -> [N / BN][K / KC][hi | lo][BN x KC canonical]; K % KC == 0, N % BN == 0
inline void pack_conv_weights(const float* w, int K, int N, float* out) {
    const int BN = tile_n(N), nk = K / KC;
    for (int nt = 0; nt < N / BN; ++nt)
        for (int kk = 0; kk < nk; ++kk) {
            float* blk = out + ((size_t)nt * nk + kk) * 2 * BN * KC;
            for (int n = 0; n < BN; ++n)
                for (int k = 0; k < KC; ++k) {
                    const float v = w[(size_t)(kk * KC + k) * N + nt * BN + n];
                    uint32_t bits;
                    memcpy(&bits, &v, 4);
                    bits &= 0xffffe000u;
                    float h;
                    memcpy(&h, &bits, 4);
                    blk[canon(n, k)] = h;
                    blk[BN * KC + canon(n, k)] = v - h;
                }
        }
}

}  // namespace rn
}  // namespace bmb
