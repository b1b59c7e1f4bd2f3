// pointwise_tc.cuh -- 1x1 convolution (GEMM) on the Hopper tensor cores: wgmma kind tf32 with a three-term split so
// that the result keeps float32 accuracy (the path's embedding bound is 1e-4):
//
//     a = a_hi + a_lo,  w = w_hi + w_lo   (hi = top 19 bits, lo = exact remainder)
//     D += A_hi*W_hi + A_hi*W_lo + A_lo*W_hi          (the dropped A_lo*W_lo term is ~2^-22 relative)
//
// One persistent CTA = 256 threads (two warpgroups): tiles of 128 output rows x all N output channels.
//   * weights (both halves, pre-arranged in the canonical K-major layout at model load) are pulled into shared memory
//     once per CTA by a bulk async copy (cp.async.bulk, completes on an mbarrier);
//   * per tile the 128 x K activation block is loaded by all threads (float4, coalesced), optionally built on the fly
//     as the gated sum of the four OSBlock branches, split into hi / lo and written in the canonical no-swizzle K-major
//     layout (8-row x 16-byte core matrices);
//   * warpgroup g issues the wgmma chain (3 per 8-wide K step) for rows 64 g .. 64 g + 63 into register accumulators;
//     its epilogue adds bias / residual, applies ReLU and stores float2 pairs.
// Layout reference: cute/atom/mma_traits_sm90_gmma.hpp (INTERLEAVE K-major canonical layout
// ((8,m),(T,2)):((1T,SBO),(1,LBO))) and cute/arch/mma_sm90_desc.hpp (descriptor bit fields).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace bmb {
namespace tc {

constexpr int TILE_M = 128;
constexpr int KC = 64;        // K chunk staged in shared memory per MMA batch (floats)
constexpr int THREADS = 256;
constexpr int NPAD_MAX = 128;   // widest accumulator (64 registers per thread)

struct Args {
    const float* in;          // PLAIN: [M][K]; GATED: x [M][K - mid] (null when K == mid)
    const float* branch[4];   // GATED: four [M][mid]
    const float* gates;       // GATED: [crops][4][mid], null for PLAIN
    const float* w_tc;        // canonical hi block then lo block, each Npad x Kpad floats
    const float* bias;        // [N]
    const float* residual;    // [M][N] or null
    float* out;               // [M][N]
    int K, N, Kpad, Npad, mid, HW, relu;
};

using um::smem_u32;

// canonical (no swizzle, K-major) offset in floats of element (row, k) in a block whose K extent is `kext`
__device__ __host__ __forceinline__ size_t canon_off(int row, int k, int kext) {
    return (size_t)(row >> 3) * ((size_t)kext * 8) + (size_t)(k >> 2) * 32 + (size_t)(row & 7) * 4 + (k & 3);
}

template <bool GATED>
__global__ void __launch_bounds__(THREADS) k_pointwise_tc(const Args a, const int* __restrict__ d_n, int off, int cap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar_w;
    int n_crops = *d_n - off;
    n_crops = n_crops < 0 ? 0 : (n_crops > cap ? cap : n_crops);
    const int M = n_crops * a.HW;
    const int n_tiles = M / TILE_M;  // HW is a multiple of 128
    if ((int)blockIdx.x >= n_tiles) return;

    const int Kpad = a.Kpad, Npad = a.Npad, K = a.K, N = a.N;
    const int kc_max = Kpad < KC ? Kpad : KC;
    float* sB = reinterpret_cast<float*>(smem_raw);                 // [2][Npad x Kpad] canonical
    float* sA_hi = sB + 2 * (size_t)Npad * Kpad;                    // [128 x kc] canonical
    float* sA_lo = sA_hi + (size_t)TILE_M * kc_max;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);

    if (threadIdx.x == 0) {
        um::mbar_init(&bar_w, 1);
        um::fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t wbytes = (uint32_t)(2 * (size_t)Npad * Kpad * sizeof(float));
        um::mbar_expect_tx(&bar_w, wbytes);
        um::bulk_g2s(sB, a.w_tc, wbytes, &bar_w);
    }
    const int KX = GATED ? K - a.mid : 0;
    bool weights_ready = false;
    float acc[2 * NPAD_MAX / 4];

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int m0 = tile * TILE_M;
        for (int k0 = 0; k0 < Kpad; k0 += KC) {
            const int kc = (Kpad - k0) < KC ? (Kpad - k0) : KC;
            // ---- stage A chunk: 128 rows x kc, float4 along k, split hi / lo, canonical layout ----
            const int f4_per_row = kc >> 2;
            for (int e = threadIdx.x; e < TILE_M * f4_per_row; e += THREADS) {
                const int r = e / f4_per_row, kq = (e - r * f4_per_row) * 4;
                const int m = m0 + r, k = k0 + kq;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (k < K) {
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
                float4 hi, lo;
                hi.x = __uint_as_float(__float_as_uint(v.x) & 0xffffe000u); lo.x = v.x - hi.x;
                hi.y = __uint_as_float(__float_as_uint(v.y) & 0xffffe000u); lo.y = v.y - hi.y;
                hi.z = __uint_as_float(__float_as_uint(v.z) & 0xffffe000u); lo.z = v.z - hi.z;
                hi.w = __uint_as_float(__float_as_uint(v.w) & 0xffffe000u); lo.w = v.w - hi.w;
                const size_t o = canon_off(r, kq, kc);
                *reinterpret_cast<float4*>(sA_hi + o) = hi;
                *reinterpret_cast<float4*>(sA_lo + o) = lo;
            }
            um::fence_async_smem();
            __syncthreads();
            // ---- MMA chain for this chunk: warpgroup wg owns rows 64 wg .. 64 wg + 63 (8 row groups of kc * 32 bytes) ----
            if (!weights_ready) { um::mbar_wait(&bar_w, 0); weights_ready = true; }
            {
                const uint32_t sbo_a = (uint32_t)kc * 32, sbo_b = (uint32_t)Kpad * 32;  // bytes between 8-row groups
                const uint32_t a_hi = smem_u32(sA_hi) + (uint32_t)wg * 8u * sbo_a, a_lo = smem_u32(sA_lo) + (uint32_t)wg * 8u * sbo_a;
                const uint32_t b_hi = smem_u32(sB), b_lo = smem_u32(sB + (size_t)Npad * Kpad);
                um::wg_fence();
                for (int ks = 0; ks < kc; ks += 8) {
                    const uint32_t ao = (uint32_t)(ks >> 2) * 128, bo = (uint32_t)((k0 + ks) >> 2) * 128;
                    const uint64_t dah = um::make_desc(a_hi + ao, 128, sbo_a), dal = um::make_desc(a_lo + ao, 128, sbo_a);
                    um::mma_rt<true>(Npad, acc, dah, b_hi + bo, 128, sbo_b, (k0 + ks) > 0 ? 1u : 0u);
                    um::mma_rt<true>(Npad, acc, dah, b_lo + bo, 128, sbo_b, 1u);
                    um::mma_rt<true>(Npad, acc, dal, b_hi + bo, 128, sbo_b, 1u);
                }
                um::wg_commit();
                um::wg_wait_all();
                um::wg_fence_acc<2 * NPAD_MAX / 4>(acc);
            }
            __syncthreads();  // both warpgroups have read the A chunk before it is restaged
        }
        // ---- epilogue: registers -> bias / residual / ReLU -> global (two rows x 2 columns per 8-column group) ----
#pragma unroll
        for (int i = 0; i < NPAD_MAX / 8; ++i) {
            const int c = 8 * i + cq;
            if (c < N) {
                const float2 b = *reinterpret_cast<const float2*>(a.bias + c);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + row + 8 * h;
                    float2 o = make_float2(acc[4 * i + 2 * h] + b.x, acc[4 * i + 2 * h + 1] + b.y);
                    if (a.residual) {
                        const float2 r = *reinterpret_cast<const float2*>(a.residual + (size_t)m * N + c);
                        o.x += r.x; o.y += r.y;
                    }
                    if (a.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                    if (a.relu == 2) { o.x = fminf(o.x, 6.f); o.y = fminf(o.y, 6.f); }
                    *reinterpret_cast<float2*>(a.out + (size_t)m * N + c) = o;
                }
            }
        }
    }
}

inline size_t smem_bytes(int Kpad, int Npad) {
    const int kc = Kpad < KC ? Kpad : KC;
    return sizeof(float) * (2 * (size_t)Npad * Kpad + 2 * (size_t)TILE_M * kc) + 128;
}

// host: arrange W[K][N] (K-major rows of N, as in the blob) into the canonical hi / lo blocks
inline void pack_weights(const float* w, int K, int N, int Kpad, int Npad, float* out /* 2*Npad*Kpad */) {
    for (size_t i = 0; i < 2 * (size_t)Npad * Kpad; ++i) out[i] = 0.f;
    for (int n = 0; n < N; ++n)
        for (int k = 0; k < K; ++k) {
            const float v = w[(size_t)k * N + n];
            uint32_t bits;
            memcpy(&bits, &v, 4);
            bits &= 0xffffe000u;
            float hi;
            memcpy(&hi, &bits, 4);
            const size_t o = canon_off(n, k, Kpad);
            out[o] = hi;
            out[(size_t)Npad * Kpad + o] = v - hi;
        }
}

}  // namespace tc
}  // namespace bmb
