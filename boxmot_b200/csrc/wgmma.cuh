// wgmma.cuh -- inline-PTX wrappers for the sm_90a tensor-core path of the ReID network: wgmma.mma_async (BF16 or TF32
// operands read from shared memory through matrix descriptors, FP32 accumulators in registers), TMA tensor loads
// (cp.async.bulk.tensor), bulk copies and mbarriers.
//
// Operand layout used everywhere ("channel-blocked planes"): element (pixel p, channel c) of an activation lives at
//     plane (c / 8), pixel p, lane (c % 8)         ->   byte offset  (c/8) * plane_stride + p * 16 + (c%8) * 2
// i.e. one 16-byte row of a core matrix per (pixel, 8-channel block); 8 consecutive pixels are one contiguous
// 128-byte core matrix.  This is the canonical no-swizzle K-major layout ((8,m),(T,2)):((1T,SBO),(1,LBO)) of
// cute/atom/mma_traits_sm90_gmma.hpp with SBO = 128 B and LBO = plane stride, so a pixel shift (a convolution tap) is a
// start-address shift of 16 B per pixel, and the same layout is what a 5-D TMA box (8, x, y, C/8, crop) writes.
// Weights use the same layout with the output channel in the pixel role.
//
// Accumulator fragment of one m64nN wgmma (thread t of the warpgroup, warp w = t / 32, lane l = t % 32): register
// d[4 i + 2 h + e] holds row 16 w + l / 4 + 8 h, column 8 i + 2 (l % 4) + e.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace bmb {
namespace um {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// bounded wait: a protocol bug must trap instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
        uint32_t done;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return;
    }
    __trap();
}

// ---- proxies / fences ----
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// ---- wgmma ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// waits until at most N committed groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across an asynchronous wgmma
template <int NREG>
__device__ __forceinline__ void wg_fence_acc(float* d) {
#pragma unroll
    for (int i = 0; i < NREG; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// GmmaDescriptor (cute/arch/mma_sm90_desc.hpp): start[0,14) | LBO[16,30) | SBO[32,46) | base offset 0 | layout 0 = no swizzle
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    return d;
}

// m64nNk16 (BF16) / m64nNk8 (TF32), both operands K-major, D (+)= A B; accumulate = 0 overwrites D
__device__ __forceinline__ void wg_bf16_n16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_bf16_n32(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_bf16_n64(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_bf16_n128(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_tf32_n16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_tf32_n32(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_tf32_n64(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wg_tf32_n128(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc));
}

// D[:, 0:N] (+)= A B[0:N] for N a multiple of 16 <= 256, issued as n128 / n64 / n32 / n16 pieces.  B is K-major with
// b_sbo bytes between groups of 8 output channels; d points at the accumulator registers of column 0.
template <int N, bool TF32>
__device__ __forceinline__ void mma(float* d, uint64_t a, uint32_t b_addr, uint32_t b_lbo, uint32_t b_sbo, uint32_t acc) {
    static_assert(N % 16 == 0 && N >= 0 && N <= 256, "N must be a multiple of 16");
    if constexpr (N >= 128) {
        if constexpr (TF32) wg_tf32_n128(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        else wg_bf16_n128(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        mma<N - 128, TF32>(d + 64, a, b_addr + 16 * b_sbo, b_lbo, b_sbo, acc);
    } else if constexpr (N >= 64) {
        if constexpr (TF32) wg_tf32_n64(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        else wg_bf16_n64(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        mma<N - 64, TF32>(d + 32, a, b_addr + 8 * b_sbo, b_lbo, b_sbo, acc);
    } else if constexpr (N >= 32) {
        if constexpr (TF32) wg_tf32_n32(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        else wg_bf16_n32(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        mma<N - 32, TF32>(d + 16, a, b_addr + 4 * b_sbo, b_lbo, b_sbo, acc);
    } else if constexpr (N >= 16) {
        if constexpr (TF32) wg_tf32_n16(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
        else wg_bf16_n16(d, a, make_desc(b_addr, b_lbo, b_sbo), acc);
    }
}
// the same with N known at run time (N in 16 .. 128, multiple of 16); d holds 64 registers.  The switch around every
// MMA makes ptxas serialise the wgmma of the caller; only the opt-in tf32 pointwise kernel uses it.
template <bool TF32>
__device__ __forceinline__ void mma_rt(int N, float* d, uint64_t a, uint32_t b_addr, uint32_t b_lbo, uint32_t b_sbo, uint32_t acc) {
    switch (N) {
        case 16: mma<16, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        case 32: mma<32, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        case 48: mma<48, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        case 64: mma<64, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        case 80: mma<80, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        case 96: mma<96, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        case 112: mma<112, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
        default: mma<128, TF32>(d, a, b_addr, b_lbo, b_sbo, acc); break;
    }
}

// named barrier over `count` threads (count a multiple of 32)
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// two-lane float arithmetic, IEEE per lane and never contracted (the depthwise walkers pair channels this way)
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, int c0, int c1, int c2, int c3, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, int c0, int c1, int c2, int c3, int c4, const void* src) {
    asm volatile(
        "cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
        ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// L2 prefetch of a 4-D box (no shared-memory destination, no barrier)
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- split-BF16 ("hi + lo") arithmetic: x ~= hi + lo with |x - hi - lo| <= 2^-17 |x| ----
// cheaper variant for the depthwise walkers: hi = the float's upper 16 bits (truncation instead of rounding: one PRMT packs
// the pair, one LOP3 per value recovers hi as a float), lo = bf16_rn(x - hi); |x - hi - lo| <= 2^-16 |x|
__device__ __forceinline__ void split2_tz(float a, float b, uint32_t& hi, uint32_t& lo) {
    const uint32_t ua = __float_as_uint(a), ub = __float_as_uint(b);
    hi = __byte_perm(ua, ub, 0x7632);                           // low half = a's upper bits, high half = b's
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(ua & 0xffff0000u), b - __uint_as_float(ub & 0xffff0000u));
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);       // .x = a (low half), .y = b
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ float2 join2(uint32_t hi, uint32_t lo) {
    const float2 h = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hi));
    const float2 l = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&lo));
    return make_float2(h.x + l.x, h.y + l.y);
}

}  // namespace um

// ---- host: 5-D tensor map over a channel-blocked activation tensor [crops][C/8][H][W][8] of BF16 ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled tensor_map_encoder();   // resolved through cudaGetDriverEntryPoint (no link-time libcuda dependency)
}  // namespace bmb
