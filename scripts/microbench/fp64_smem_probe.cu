// Probe of the primitives the one-CTA-per-stream float64 kernels are made of (dense JV solver, Kalman update):
// FP64 add latency / throughput, shared-memory pointer-chase latency through a typed (LDS) and a generic (LD.E)
// pointer, and the cost of __syncthreads_or, all for ONE CTA of 256 threads on one SM -- the launch shape of
// k_docs_frame.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_smem_probe fp64_smem_probe.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_dadd_latency(double* out, long long* cyc, int n, double a) {
    double x = out[threadIdx.x];
    const long long t0 = clock64();
    for (int i = 0; i < n; ++i) x = x + a;   // dependent chain
    const long long t1 = clock64();
    out[threadIdx.x] = x;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void k_dadd_throughput(double* out, long long* cyc, int n, double a) {
    double x0 = out[threadIdx.x], x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < n; ++i) { x0 += a; x1 += a; x2 += a; x3 += a; x4 += a; x5 += a; x6 += a; x7 += a; }
    __syncthreads();
    const long long t1 = clock64();
    out[threadIdx.x] = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void k_fadd_throughput(float* out, long long* cyc, int n, float a) {
    float x0 = out[threadIdx.x], x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < n; ++i) { x0 += a; x1 += a; x2 += a; x3 += a; x4 += a; x5 += a; x6 += a; x7 += a; }
    __syncthreads();
    const long long t1 = clock64();
    out[threadIdx.x] = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void k_dsetp_chain(double* out, long long* cyc, int n, double a) {
    // relax-like body: r = nv - h; if (r < d) d = r;   (DADD + DSETP + select), 8 independent columns
    double d[8], nv[8];
    for (int q = 0; q < 8; ++q) { d[q] = out[threadIdx.x] + q; nv[q] = d[q] * 0.5; }
    double h = a;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < n; ++i) {
#pragma unroll
        for (int q = 0; q < 8; ++q) { const double r = nv[q] - h; if (r < d[q]) d[q] = r; }
        h += 1e-3;
    }
    __syncthreads();
    const long long t1 = clock64();
    double s = 0;
    for (int q = 0; q < 8; ++q) s += d[q];
    out[threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void k_chase(const int* init, int* sink, long long* cyc, int n, int generic, int* gbuf) {
    __shared__ int arr[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) arr[i] = init[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        const int* p = generic == 0 ? arr : (generic == 1 ? (const int*)arr : gbuf);
        // generic == 1: launder the pointer through global memory so the compiler loses the address space
        if (generic == 1) { ((const int**)sink)[1] = arr; __threadfence(); p = ((const int* volatile*)sink)[1]; }
        int idx = 0;
        long long t0, t1;
        if (generic == 0) {
            t0 = clock64();
            for (int i = 0; i < n; ++i) idx = arr[idx];
            t1 = clock64();
        } else {
            t0 = clock64();
            for (int i = 0; i < n; ++i) idx = p[idx];
            t1 = clock64();
        }
        sink[0] = idx;
        cyc[0] = t1 - t0;
    }
}

__global__ void k_barrier(int* sink, long long* cyc, int n) {
    int acc = 0;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < n; ++i) acc += __syncthreads_or((threadIdx.x == (unsigned)(i & 255)) && (i & 1023) == 1023);
    const long long t1 = clock64();
    if (threadIdx.x == 0) { sink[0] = acc; cyc[0] = t1 - t0; }
}

#define OK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

int main() {
    double* dout; float* fout; long long* cyc; int *init, *sink, *gbuf;
    OK(cudaMalloc(&dout, 8 * 1024)); OK(cudaMalloc(&fout, 4 * 1024)); OK(cudaMalloc(&cyc, 64));
    OK(cudaMalloc(&init, 4 * 1024)); OK(cudaMalloc(&sink, 64)); OK(cudaMalloc(&gbuf, 4 * 1024));
    OK(cudaMemset(dout, 0, 8 * 1024)); OK(cudaMemset(fout, 0, 4 * 1024));
    int h[1024];
    for (int i = 0; i < 1024; ++i) h[i] = (i * 37 + 11) & 1023;   // a permutation walk
    OK(cudaMemcpy(init, h, sizeof h, cudaMemcpyHostToDevice)); OK(cudaMemcpy(gbuf, h, sizeof h, cudaMemcpyHostToDevice));
    long long c = 0;
    const int N = 4096;
    auto rd = [&]() { cudaDeviceSynchronize(); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost); return (double)c; };
    for (int rep = 0; rep < 2; ++rep) {   // second pass is warm
        k_dadd_latency<<<1, 32>>>(dout, cyc, N, 1e-9);            const double a = rd() / N;
        k_dadd_throughput<<<1, 256>>>(dout, cyc, N, 1e-9);        const double b = rd() / N;   // 8 DADD per thread per iter
        k_fadd_throughput<<<1, 256>>>(fout, cyc, N, 1e-9f);       const double b2 = rd() / N;
        k_dsetp_chain<<<1, 256>>>(dout, cyc, N, 1e-9);            const double d = rd() / N;
        k_chase<<<1, 256>>>(init, sink, cyc, N, 0, gbuf);         const double e0 = rd() / N;
        k_chase<<<1, 256>>>(init, sink, cyc, N, 1, gbuf);         const double e1 = rd() / N;
        k_chase<<<1, 256>>>(init, sink, cyc, N, 2, gbuf);         const double e2 = rd() / N;
        k_barrier<<<1, 256>>>(sink, cyc, N);                      const double f = rd() / N;
        if (rep)
            printf("{\"dadd_latency_cycles\": %.1f, \"dadd_8x256thr_cycles_per_iter\": %.1f, \"fadd_8x256thr_cycles_per_iter\": %.1f, "
                   "\"relax8_256thr_cycles_per_iter\": %.1f, \"lds_chase_cycles\": %.1f, \"generic_smem_chase_cycles\": %.1f, "
                   "\"global_l1_chase_cycles\": %.1f, \"syncthreads_or_256thr_cycles\": %.1f}\n", a, b, b2, d, e0, e1, e2, f);
    }
    OK(cudaGetLastError());
    return 0;
}
