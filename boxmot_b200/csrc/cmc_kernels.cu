// cmc_kernels.cu -- launchers of the on-device ECC camera-motion estimator (cmc_ecc.cuh; SURVEY 8f-3).
// Built with -fmad=false like the other tracker translation units: the float32 image arithmetic follows OpenCV's
// operation order.
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>
#include <vector>

#include "cmc_ecc.cuh"
#include "engine.h"

namespace bmb {

#define CMC_CUDA_OK(x)                                                                                              \
    do {                                                                                                            \
        cudaError_t e_ = (x);                                                                                       \
        if (e_ != cudaSuccess) throw std::runtime_error(std::string("CUDA: ") + cudaGetErrorString(e_) + " at " #x); \
    } while (0)

// BaseCMC.preprocess for every stream: one thread per pixel of the registration image (4 BGR source pixels each)
__global__ void __launch_bounds__(256) k_cmc_prepare(const uint8_t* images, size_t image_stride, int rows, int cols,
                                                     double inv_scale, uint8_t* cur, int h, int w) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= h * w) return;
    const int s = blockIdx.y;
    const int y = p / w, x = p - y * w;
    cur[(size_t)s * h * w + p] = cmc_prepare_pixel(images + image_stride * s, rows, cols, inv_scale, y, x);
}

// ECC.apply for every stream (one CTA each): estimate the translation prev -> cur, publish it as the stream's pending
// 2x3 warp (what set_warp would have written), then cur becomes prev.  `gate[s]` (may be null) points at a device count:
// the stream is skipped while it is zero -- StrongSORT only calls apply() on frames that start with at least one track
// (strongsort.py:83-86), so its previous image is the last frame that had tracks.
__global__ void __launch_bounds__(512) k_cmc_ecc(uint8_t* prev, const uint8_t* cur, int* has_prev, const int* const* gate,
                                                 int h, int w, double eps, int max_iter, float scale, double* warp) {
    __shared__ double red[16 * 8];
    const int s = blockIdx.x;
    if (gate && gate[s] && *gate[s] < 1) return;
    uint8_t* T = prev + (size_t)s * h * w;
    const uint8_t* I = cur + (size_t)s * h * w;
    const bool hp = has_prev[s] != 0;
    float txy[2] = {0.f, 0.f};
    int status = 1;
    if (hp) status = ecc_translation(T, I, h, w, eps, max_iter, red, txy);
    if (threadIdx.x == 0) {
        double* wp = warp + (size_t)s * 8;
        const bool ok = hp && status == 0;
        // `warp_matrix[0, 2] /= self.scale` on a float32 matrix (ecc.py:83-86); identity when there is no previous image
        // or OpenCV would have raised StsNoConv
        const float fx = ok ? (scale < 1.0f ? txy[0] / scale : txy[0]) : 0.f;
        const float fy = ok ? (scale < 1.0f ? txy[1] / scale : txy[1]) : 0.f;
        wp[0] = 1.0; wp[1] = 0.0; wp[2] = (double)fx;
        wp[3] = 0.0; wp[4] = 1.0; wp[5] = (double)fy;
        wp[6] = ok ? 1.0 : 0.0;   // pending flag; an identity needs no application (exact no-op in the trackers)
        wp[7] = 0.0;
    }
    __syncthreads();   // every thread is done reading the template
    for (int p = threadIdx.x; p < h * w; p += blockDim.x) T[p] = I[p];
    if (threadIdx.x == 0) has_prev[s] = 1;
}

void cmc_enqueue_prepare(const uint8_t* images, size_t image_stride, int rows, int cols, int S, double scale, uint8_t* out,
                         cudaStream_t st) {
    int h, w;
    cmc_scaled_size(rows, cols, scale, &h, &w);
    dim3 g((h * w + 255) / 256, S);
    k_cmc_prepare<<<g, 256, 0, st>>>(images, image_stride, rows, cols, 1.0 / scale, out, h, w);
}

void cmc_enqueue_ecc(const uint8_t* images, size_t image_stride, int rows, int cols, int S, double scale, double eps,
                     int max_iter, uint8_t* prev, uint8_t* cur, int* has_prev, const int* const* gate, double* warp,
                     cudaStream_t st) {
    int h, w;
    cmc_scaled_size(rows, cols, scale, &h, &w);
    cmc_enqueue_prepare(images, image_stride, rows, cols, S, scale, cur, st);
    k_cmc_ecc<<<S, 512, 0, st>>>(prev, cur, has_prev, gate, h, w, eps, max_iter, (float)scale, warp);
    CMC_CUDA_OK(cudaGetLastError());
}

// ECC().apply(prev_bgr) then ECC().apply(cur_bgr): the float32 2x3 warp of the second call, for parity tests.
// status: 0 estimated, 1 OpenCV would have raised StsNoConv (identity returned).
void standalone_ecc(const uint8_t* prev_bgr, const uint8_t* cur_bgr, int rows, int cols, double scale, double eps,
                    int max_iter, float* warp6, int* status, uint8_t* prepared_out) {
    if (rows < 8 || cols < 8 || !(scale > 0.0)) throw std::runtime_error("cmc: bad frame size / scale");
    int h, w;
    cmc_scaled_size(rows, cols, scale, &h, &w);
    if (h < 3 || w < 3) throw std::runtime_error("cmc: registration image smaller than 3x3");
    const size_t ib = (size_t)rows * cols * 3, sb = (size_t)h * w;
    uint8_t *d_img = nullptr, *d_prev = nullptr, *d_cur = nullptr;
    int* d_has = nullptr;
    double* d_warp = nullptr;
    try {
        CMC_CUDA_OK(cudaMalloc(&d_img, ib));
        CMC_CUDA_OK(cudaMalloc(&d_prev, sb));
        CMC_CUDA_OK(cudaMalloc(&d_cur, sb));
        CMC_CUDA_OK(cudaMalloc(&d_has, sizeof(int)));
        CMC_CUDA_OK(cudaMalloc(&d_warp, sizeof(double) * 8));
        CMC_CUDA_OK(cudaMemset(d_has, 0, sizeof(int)));
        double w8[8];
        for (int f = 0; f < 2; ++f) {
            CMC_CUDA_OK(cudaMemcpy(d_img, f ? cur_bgr : prev_bgr, ib, cudaMemcpyHostToDevice));
            cmc_enqueue_ecc(d_img, ib, rows, cols, 1, scale, eps, max_iter, d_prev, d_cur, d_has, nullptr, d_warp, 0);
            CMC_CUDA_OK(cudaDeviceSynchronize());
        }
        CMC_CUDA_OK(cudaMemcpy(w8, d_warp, sizeof(w8), cudaMemcpyDeviceToHost));
        for (int k = 0; k < 6; ++k) warp6[k] = (float)w8[k];
        if (status) *status = w8[6] != 0.0 ? 0 : 1;
        if (prepared_out) CMC_CUDA_OK(cudaMemcpy(prepared_out, d_cur, sb, cudaMemcpyDeviceToHost));
    } catch (...) {
        cudaFree(d_img); cudaFree(d_prev); cudaFree(d_cur); cudaFree(d_has); cudaFree(d_warp);
        throw;
    }
    cudaFree(d_img); cudaFree(d_prev); cudaFree(d_cur); cudaFree(d_has); cudaFree(d_warp);
}

}  // namespace bmb
