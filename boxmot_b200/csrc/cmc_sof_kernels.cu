// cmc_sof_kernels.cu -- launchers of the on-device SOF camera-motion estimator (cmc_sof.cuh), batched over S streams.
// Built with -fmad=false like the other tracker translation units: the float32 image arithmetic follows OpenCV's
// operation order, and the host build of cmc_sof.cuh (tests/_sofsim) must give the same bits.
//
// One frame is eleven launches; every kernel reads the stream's `initialized` flag and skips the work SOF.apply would not
// do on that frame (cornerSubPix only initialises, LK / RANSAC only track):
//   prepare (BaseCMC.preprocess) -> mask + Sobel + level-0 Scharr -> eigenvalue map + masked max -> candidates ->
//   pyramid levels 1.. -> top-1000 selection -> cornerSubPix -> LK (one warp per point) -> RANSAC draws + models ->
//   RANSAC scores (one warp per hypothesis) -> pick + refine + decision + state update.
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>

#include "cmc_sof.cuh"
#include "engine.h"

namespace bmb {

#define SOF_CUDA_OK(x)                                                                                              \
    do {                                                                                                            \
        cudaError_t e_ = (x);                                                                                       \
        if (e_ != cudaSuccess) throw std::runtime_error(std::string("CUDA: ") + cudaGetErrorString(e_) + " at " #x); \
    } while (0)

namespace {

constexpr int K2 = 2 * SOF_MAX_CORNERS;   // floats of one keypoint list

// per-stream device buffers; `pyr[cur]` / `der[cur]` receive this frame, the other pair holds the previous frame
struct SofBufs {
    uint8_t* gray;      // [S][h*w]
    uint8_t* pyr[2];    // [S][npx]
    int16_t* der[2];    // [S][2*npx]
    uint8_t* mask;      // [S][h*w]
    float* sob;         // [S][2][h*w]
    float* eig;         // [S][h*w]
    unsigned* maxkey;   // [S]
    unsigned long long* cand;   // [S][h*w]
    int* ncand;         // [S]
    float* corners;     // [S][K2]
    int* ncorners;      // [S]
    float* prev_kps;    // [S][K2]
    int* nprev;         // [S]
    int* initialized;   // [S]
    float* next;        // [S][K2]
    int* lkst;          // [S][SOF_MAX_CORNERS]
    float* pv;          // [S][K2]
    float* nv;          // [S][K2]
    int* nvalid;        // [S]
    int* pairs;         // [S][2*SOF_RANSAC_ITERS]
    double* models;     // [S][6*SOF_RANSAC_ITERS]
    int* good;          // [S][SOF_RANSAC_ITERS]
    float* warp;        // [S][6]
    int* status;        // [S]
};

}  // namespace

// the detection rows whose boxes are cleared from the corner mask: [S][cap][stride] floats, n[S] rows per stream
struct SofDets {
    const float* rows;
    const int* n;
    int cap, stride, conf_col;
    float conf_thr;
};

namespace {

__global__ void __launch_bounds__(256) k_sof_level0(SofBufs b, int cur, SofGeom g, SofDets dt, float scale) {
    const int h = g.h, w = g.w, p = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
    if (p >= h * w) return;
    const int y = p / w, x = p - y * w;
    const uint8_t* gray = b.gray + (size_t)s * h * w;
    b.pyr[cur][(size_t)s * g.npx + p] = gray[p];
    b.mask[(size_t)s * h * w + p] = sof_mask_pixel(h, w, y, x, dt.rows + (size_t)s * dt.cap * dt.stride, dt.n[s], dt.stride,
                                                   scale, dt.conf_col, dt.conf_thr);
    float dx, dy;
    sof_sobel(gray, h, w, y, x, dx, dy);
    b.sob[(size_t)s * 2 * h * w + p] = dx;
    b.sob[(size_t)s * 2 * h * w + h * w + p] = dy;
    sof_scharr_pixel(gray, h, w, y, x, b.der[cur] + (size_t)s * 2 * g.npx + 2 * p);
}

__global__ void __launch_bounds__(256) k_sof_eig(SofBufs b, int h, int w) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
    if (p >= h * w) return;
    const float* sob = b.sob + (size_t)s * 2 * h * w;
    const float e = sof_eig_pixel(sob, sob + h * w, h, w, p / w, p % w);
    b.eig[(size_t)s * h * w + p] = e;
    if (b.mask[(size_t)s * h * w + p]) atomicMax(b.maxkey + s, sof_fkey(e));   // exact: any order gives the same max
}

__device__ float sof_unkey(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(256) k_sof_candidates(SofBufs b, int h, int w) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
    if (p >= h * w) return;
    const unsigned mk = b.maxkey[s];
    const float mx = mk ? sof_unkey(mk) : 0.f;   // minMaxLoc over an empty mask reports 0
    const float thr = (float)((double)mx * 0.01);
    const unsigned long long k = sof_candidate(b.eig + (size_t)s * h * w, b.mask + (size_t)s * h * w, h, w, p / w, p % w, thr);
    if (k) b.cand[(size_t)s * h * w + atomicAdd(b.ncand + s, 1)] = k;   // order restored by the key sort
}

// pyramid levels 1.. of this frame and their Scharr derivatives: one CTA per stream, one level after the other
__global__ void __launch_bounds__(1024) k_sof_pyramid(SofBufs b, int cur, SofGeom g) {
    const int s = blockIdx.x;
    uint8_t* P = b.pyr[cur] + (size_t)s * g.npx;
    int16_t* D = b.der[cur] + (size_t)s * 2 * g.npx;
    for (int l = 1; l < g.nlev; ++l) {
        const int n = g.lh[l] * g.lw[l];
        for (int p = threadIdx.x; p < n; p += blockDim.x)
            P[g.off[l] + p] = sof_pyrdown_pixel(P + g.off[l - 1], g.lh[l - 1], g.lw[l - 1], p / g.lw[l], p % g.lw[l]);
        __syncthreads();
        for (int p = threadIdx.x; p < n; p += blockDim.x)
            sof_scharr_pixel(P + g.off[l], g.lh[l], g.lw[l], p / g.lw[l], p % g.lw[l], D + 2 * ((size_t)g.off[l] + p));
        __syncthreads();
    }
}

// goodFeaturesToTrack's sort and cut: the 1000th largest key by an 8-bit radix select (when there are more), then the
// at most 1000 kept keys ranked by counting.  Keys are unique (they carry the address), so the result is the sorted
// list whatever order the candidates were compacted in.
__global__ void __launch_bounds__(1024) k_sof_select(SofBufs b, int h, int w) {
    __shared__ unsigned hist[256];
    __shared__ unsigned long long keep[SOF_MAX_CORNERS];
    __shared__ unsigned long long s_prefix, s_mask;
    __shared__ int s_want, s_nkeep;
    const int s = blockIdx.x, t = threadIdx.x;
    const int n = b.ncand[s];
    const unsigned long long* K = b.cand + (size_t)s * h * w;
    if (t == 0) { s_prefix = 0; s_mask = 0; s_want = SOF_MAX_CORNERS; s_nkeep = 0; }
    __syncthreads();
    unsigned long long kth = 0;   // keys >= kth are kept
    if (n > SOF_MAX_CORNERS) {
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int i = t; i < 256; i += blockDim.x) hist[i] = 0;
            __syncthreads();
            const unsigned long long pre = s_prefix, msk = s_mask;
            for (int i = t; i < n; i += blockDim.x)
                if ((K[i] & msk) == pre) atomicAdd(&hist[(K[i] >> shift) & 255], 1u);
            __syncthreads();
            if (t == 0) {
                int want = s_want, d = 255;
                for (; d > 0 && (int)hist[d] < want; --d) want -= hist[d];
                s_want = want;
                s_prefix = pre | ((unsigned long long)d << shift);
                s_mask = msk | (255ull << shift);
            }
            __syncthreads();
        }
        kth = s_prefix;
    }
    for (int i = t; i < n; i += blockDim.x)
        if (K[i] >= kth) keep[atomicAdd(&s_nkeep, 1)] = K[i];
    __syncthreads();
    const int m = s_nkeep;
    for (int i = t; i < m; i += blockDim.x) {
        const unsigned long long k = keep[i];
        int r = 0;
        for (int j = 0; j < m; ++j) r += keep[j] > k;
        sof_key_point(k, w, b.corners + (size_t)s * K2 + 2 * r);
    }
    if (t == 0) { b.ncorners[s] = m; b.ncand[s] = 0; b.maxkey[s] = 0; }   // ready for the next frame
}

__global__ void __launch_bounds__(128) k_sof_subpix(SofBufs b, int h, int w) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
    const int nc = b.ncorners[s];
    if (b.initialized[s] || nc < 4 || i >= nc) return;
    sof_subpix_point(b.gray + (size_t)s * h * w, h, w, b.corners + (size_t)s * K2 + 2 * i);
}

__global__ void __launch_bounds__(256) k_sof_lk(SofBufs b, int cur, SofGeom g) {
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), s = blockIdx.y;
    if (!b.initialized[s] || i >= b.nprev[s]) return;   // warp-uniform
    const float* kp = b.prev_kps + (size_t)s * K2 + 2 * i;
    float out[2];
    int st;
    sof_lk_point(g, b.pyr[cur ^ 1] + (size_t)s * g.npx, b.der[cur ^ 1] + (size_t)s * 2 * g.npx, b.pyr[cur] + (size_t)s * g.npx,
                 kp[0], kp[1], out, &st);
    if ((threadIdx.x & 31) == 0) {
        b.next[(size_t)s * K2 + 2 * i] = out[0];
        b.next[(size_t)s * K2 + 2 * i + 1] = out[1];
        b.lkst[(size_t)s * SOF_MAX_CORNERS + i] = st;
    }
}

// the tracked pairs in point order (status 1), the RANSAC index pairs (one thread) and the 2000 candidate models
__global__ void __launch_bounds__(1024) k_sof_ransac_prep(SofBufs b) {
    __shared__ int wsum[32];
    const int s = blockIdx.x, t = threadIdx.x, lane = t & 31, wp = t >> 5;
    if (!b.initialized[s]) return;
    const int np = b.nprev[s];
    const bool ok = t < np && b.lkst[(size_t)s * SOF_MAX_CORNERS + t] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wsum[wp] = __popc(bal);
    __syncthreads();
    int base = 0, total = 0;
    for (int k = 0; k < 32; ++k) { base += k < wp ? wsum[k] : 0; total += wsum[k]; }
    if (ok) {
        const int pos = base + __popc(bal & ((1u << lane) - 1u));
        const float* kp = b.prev_kps + (size_t)s * K2 + 2 * t;
        const float* nx = b.next + (size_t)s * K2 + 2 * t;
        b.pv[(size_t)s * K2 + 2 * pos] = kp[0]; b.pv[(size_t)s * K2 + 2 * pos + 1] = kp[1];
        b.nv[(size_t)s * K2 + 2 * pos] = nx[0]; b.nv[(size_t)s * K2 + 2 * pos + 1] = nx[1];
    }
    if (t == 0) b.nvalid[s] = total;
    if (total < 4) return;   // block-uniform
    int* pairs = b.pairs + (size_t)s * 2 * SOF_RANSAC_ITERS;
    if (t == 0) sof_draw_pairs(total, SOF_RANSAC_ITERS, pairs);
    __syncthreads();
    const float* pv = b.pv + (size_t)s * K2;
    const float* nv = b.nv + (size_t)s * K2;
    for (int it = t; it < SOF_RANSAC_ITERS; it += blockDim.x) {
        const int i0 = pairs[2 * it], i1 = pairs[2 * it + 1];
        sof_model(pv + 2 * i0, pv + 2 * i1, nv + 2 * i0, nv + 2 * i1, b.models + (size_t)s * 6 * SOF_RANSAC_ITERS + 6 * it);
    }
}

__global__ void __launch_bounds__(256) k_sof_ransac_score(SofBufs b, float thr2) {
    const int it = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), s = blockIdx.y, lane = threadIdx.x & 31;
    if (!b.initialized[s] || it >= SOF_RANSAC_ITERS) return;
    const int n = b.nvalid[s];
    if (n < 4) return;
    const double* M = b.models + (size_t)s * 6 * SOF_RANSAC_ITERS + 6 * it;
    const float* pv = b.pv + (size_t)s * K2;
    const float* nv = b.nv + (size_t)s * K2;
    int c = 0;
    for (int i = lane; i < n; i += 32) c += sof_inlier(M, pv + 2 * i, nv + 2 * i, thr2);
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) b.good[(size_t)s * SOF_RANSAC_ITERS + it] = c;
}

// SOF.apply's decisions for one stream (SOF_RED threads): RANSAC's pick, refine, inlier gate, returned warp, state
__global__ void __launch_bounds__(SOF_RED) k_sof_finish(SofBufs b, float thr2, float scale, int min_inliers,
                                                        double min_ratio, double* warp8) {
    __shared__ double red[6 * SOF_RED];
    __shared__ float isrc[K2], idst[K2];
    __shared__ double M[6];
    __shared__ int s_best, s_ninl;
    const int s = blockIdx.x, t = threadIdx.x;
    const int nc = b.ncorners[s];
    const float* keep = b.corners + (size_t)s * K2;   // the keypoints the next frame tracks
    int nkeep = nc, st = SOF_REJECTED;
    float w6[6] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f};
    int init_next = nc >= 4;
    const bool tracking = b.initialized[s] != 0;   // read once: thread 0 rewrites it below
    if (!tracking) {
        st = SOF_INIT;
    } else if (b.nvalid[s] >= 4) {   // otherwise SOF._reset: the fresh corners, initialised when >= 4
        const int n = b.nvalid[s];
        const float* pv = b.pv + (size_t)s * K2;
        const float* nv = b.nv + (size_t)s * K2;
        if (t == 0) {
            int bg;
            s_best = sof_ransac_pick(b.good + (size_t)s * SOF_RANSAC_ITERS, n, &bg);
            s_ninl = 0;
            if (s_best >= 0) {
                for (int k = 0; k < 6; ++k) M[k] = b.models[(size_t)s * 6 * SOF_RANSAC_ITERS + 6 * s_best + k];
                for (int i = 0; i < n; ++i)
                    if (sof_inlier(M, pv + 2 * i, nv + 2 * i, thr2)) {
                        isrc[2 * s_ninl] = pv[2 * i]; isrc[2 * s_ninl + 1] = pv[2 * i + 1];
                        idst[2 * s_ninl] = nv[2 * i]; idst[2 * s_ninl + 1] = nv[2 * i + 1];
                        ++s_ninl;
                    }
            }
        }
        __syncthreads();
        if (s_best >= 0 && sof_accept(s_ninl, n, min_inliers, min_ratio)) {
            double m[6];
            for (int k = 0; k < 6; ++k) m[k] = M[k];
            sof_refine(isrc, idst, s_ninl, m, red);
            sof_warp_out(m, scale, w6);
            st = SOF_ESTIMATED;
        }
        if (nc < 4) { keep = nv; nkeep = n; }   // re-detection found too few: keep the tracked points
        init_next = 1;
    }
    float* dst = b.prev_kps + (size_t)s * K2;
    for (int k = t; k < 2 * nkeep; k += blockDim.x) dst[k] = keep[k];
    __syncthreads();   // every thread has read this frame's state before it is replaced
    if (t == 0) {
        b.nprev[s] = nkeep;
        b.initialized[s] = init_next;
        for (int k = 0; k < 6; ++k) b.warp[6 * s + k] = w6[k];
        b.status[s] = st;
        if (warp8) {   // the tracker's pending warp (what set_warp writes); an identity is no correction at all
            double* wp = warp8 + (size_t)8 * s;
            for (int k = 0; k < 6; ++k) wp[k] = (double)w6[k];
            wp[6] = st == SOF_ESTIMATED ? 1.0 : 0.0;
            wp[7] = 0.0;
        }
    }
}

template <class T>
void sof_alloc(T*& p, size_t n) {
    SOF_CUDA_OK(cudaMalloc(&p, n * sizeof(T)));
    SOF_CUDA_OK(cudaMemset(p, 0, n * sizeof(T)));
}

}  // namespace

struct SofState {
    int S = 0, h = 0, w = 0, cur = 0, det_cap = 0;
    SofGeom g{};
    SofBufs b{};
    float* dets = nullptr;   // [S][det_cap][4]
    int* ndets = nullptr;    // [S]
    double scale;
    int min_inliers;
    double min_ratio;
    float thr;

    void free_bufs() {
        void* ps[] = {b.gray, b.pyr[0], b.pyr[1], b.der[0], b.der[1], b.mask, b.sob, b.eig, b.maxkey, b.cand, b.ncand,
                      b.corners, b.ncorners, b.prev_kps, b.nprev, b.initialized, b.next, b.lkst, b.pv, b.nv, b.nvalid,
                      b.pairs, b.models, b.good, b.warp, b.status};
        for (void* p : ps) cudaFree(p);
        b = SofBufs{};
        h = w = 0;
    }
    // the workspace follows the registration image; a new resolution starts every stream afresh
    void ensure(int hh, int ww) {
        if (hh == h && ww == w) return;
        free_bufs();
        cur = 0;
        g = sof_geom(hh, ww);
        const size_t px = (size_t)hh * ww;
        try {
            alloc_bufs(px);
        } catch (...) {
            free_bufs();   // leaves h = w = 0: the next frame allocates again
            throw;
        }
        h = hh; w = ww;
    }
    void alloc_bufs(size_t px) {
        sof_alloc(b.gray, S * px);
        for (int k = 0; k < 2; ++k) { sof_alloc(b.pyr[k], S * (size_t)g.npx); sof_alloc(b.der[k], 2 * S * (size_t)g.npx); }
        sof_alloc(b.mask, S * px);
        sof_alloc(b.sob, 2 * S * px);
        sof_alloc(b.eig, S * px);
        sof_alloc(b.maxkey, S);
        sof_alloc(b.cand, S * px);
        sof_alloc(b.ncand, S);
        sof_alloc(b.corners, S * (size_t)K2);
        sof_alloc(b.ncorners, S);
        sof_alloc(b.prev_kps, S * (size_t)K2);
        sof_alloc(b.nprev, S);
        sof_alloc(b.initialized, S);
        sof_alloc(b.next, S * (size_t)K2);
        sof_alloc(b.lkst, S * (size_t)SOF_MAX_CORNERS);
        sof_alloc(b.pv, S * (size_t)K2);
        sof_alloc(b.nv, S * (size_t)K2);
        sof_alloc(b.nvalid, S);
        sof_alloc(b.pairs, 2 * S * (size_t)SOF_RANSAC_ITERS);
        sof_alloc(b.models, 6 * S * (size_t)SOF_RANSAC_ITERS);
        sof_alloc(b.good, S * (size_t)SOF_RANSAC_ITERS);
        sof_alloc(b.warp, 6 * (size_t)S);
        sof_alloc(b.status, S);
    }
    // SOF freshly constructed for every stream (the next frame initialises)
    void reset(cudaStream_t cs) {
        if (b.initialized) SOF_CUDA_OK(cudaMemsetAsync(b.initialized, 0, sizeof(int) * S, cs));
    }
    void ensure_dets(int cap) {
        if (cap <= det_cap) return;
        cudaFree(dets);
        dets = nullptr;
        det_cap = cap;
        sof_alloc(dets, (size_t)S * cap * 4);
    }
    ~SofState() {
        free_bufs();
        cudaFree(dets);
        cudaFree(ndets);
    }
};

// SOF.apply for S streams: `images` (device, image_stride bytes apart) are BGR rows x cols; `dt` are the detection rows
// whose boxes leave the corner mask.  Results land in st.b.warp / st.b.status and, when `warp8` is given, in the
// trackers' pending-warp slots [S][8].  Returns the number of launches.
int sof_enqueue(SofState& st, const uint8_t* images, size_t image_stride, int rows, int cols, const SofDets& dt,
                double* warp8, cudaStream_t cs) {
    int h, w;
    cmc_scaled_size(rows, cols, st.scale, &h, &w);
    st.ensure(h, w);
    const int S = st.S, npx = h * w;
    const float fscale = (float)st.scale, thr2 = (float)((double)st.thr * (double)st.thr);
    cmc_enqueue_prepare(images, image_stride, rows, cols, S, st.scale, st.b.gray, cs);
    const dim3 gp((npx + 255) / 256, S);
    k_sof_level0<<<gp, 256, 0, cs>>>(st.b, st.cur, st.g, dt, fscale);
    k_sof_eig<<<gp, 256, 0, cs>>>(st.b, h, w);
    k_sof_candidates<<<gp, 256, 0, cs>>>(st.b, h, w);
    k_sof_pyramid<<<S, 1024, 0, cs>>>(st.b, st.cur, st.g);
    k_sof_select<<<S, 1024, 0, cs>>>(st.b, h, w);
    k_sof_subpix<<<dim3((SOF_MAX_CORNERS + 127) / 128, S), 128, 0, cs>>>(st.b, h, w);
    k_sof_lk<<<dim3((SOF_MAX_CORNERS + 7) / 8, S), 256, 0, cs>>>(st.b, st.cur, st.g);
    k_sof_ransac_prep<<<S, 1024, 0, cs>>>(st.b);
    k_sof_ransac_score<<<dim3(SOF_RANSAC_ITERS / 8, S), 256, 0, cs>>>(st.b, thr2);
    k_sof_finish<<<S, SOF_RED, 0, cs>>>(st.b, thr2, fscale, st.min_inliers, st.min_ratio, warp8);
    SOF_CUDA_OK(cudaGetLastError());
    st.cur ^= 1;
    return 11;
}

SofState* sof_state_create(int S, double scale, int min_inliers, double min_ratio, double thr) {
    if (S < 1 || !(scale > 0.0) || min_inliers < 0 || !(thr > 0.0)) throw std::runtime_error("cmc_sof: bad parameters");
    SofState* st = new SofState();
    st->S = S;
    st->scale = scale;
    st->min_inliers = min_inliers;
    st->min_ratio = min_ratio;
    st->thr = (float)thr;
    return st;
}
void sof_state_free(SofState* st) { delete st; }
void sof_state_reset(SofState* st, cudaStream_t cs) { st->reset(cs); }
int sof_state_enqueue(SofState* st, const uint8_t* images, size_t image_stride, int rows, int cols, const float* dets,
                      const int* ndets, int det_cap, int det_stride, int conf_col, float conf_thr, double* warp8,
                      cudaStream_t cs) {
    const SofDets dt{dets, ndets, det_cap, det_stride, conf_col, conf_thr};
    return sof_enqueue(*st, images, image_stride, rows, cols, dt, warp8, cs);
}

// ---- standalone estimator (boxmot_b200_cmc_sof_*) ------------------------------------------------------------------
struct SofHandle {
    SofState st;
    uint8_t* d_img = nullptr;
    size_t img_bytes = 0;
};

void* sof_create(double scale, int min_inliers, double min_ratio, double thr) {
    if (!(scale > 0.0) || min_inliers < 0 || !(thr > 0.0)) throw std::runtime_error("cmc_sof: bad parameters");
    SofHandle* hd = new SofHandle();
    hd->st.S = 1;
    hd->st.scale = scale;
    hd->st.min_inliers = min_inliers;
    hd->st.min_ratio = min_ratio;
    hd->st.thr = (float)thr;
    try {
        sof_alloc(hd->st.ndets, 1);
        hd->st.ensure_dets(64);
    } catch (...) {
        delete hd;
        throw;
    }
    return hd;
}

void sof_destroy(void* p) {
    SofHandle* hd = (SofHandle*)p;
    if (!hd) return;
    cudaFree(hd->d_img);
    delete hd;
}

void sof_apply(void* p, const uint8_t* bgr, int rows, int cols, const float* dets_xyxy, int n_dets, float* warp6,
               int* status) {
    SofHandle& hd = *(SofHandle*)p;
    int h, w;
    cmc_scaled_size(rows, cols, hd.st.scale, &h, &w);
    if (rows < 1 || cols < 1 || h < 3 || w < 3) throw std::runtime_error("cmc_sof: registration image smaller than 3x3");
    if (n_dets < 0 || (n_dets > 0 && !dets_xyxy)) throw std::runtime_error("cmc_sof: bad detections");
    const size_t ib = (size_t)rows * cols * 3;
    if (ib > hd.img_bytes) {
        cudaFree(hd.d_img);
        hd.d_img = nullptr;
        hd.img_bytes = 0;
        SOF_CUDA_OK(cudaMalloc(&hd.d_img, ib));
        hd.img_bytes = ib;
    }
    hd.st.ensure_dets(n_dets);
    SOF_CUDA_OK(cudaMemcpy(hd.d_img, bgr, ib, cudaMemcpyHostToDevice));
    if (n_dets) SOF_CUDA_OK(cudaMemcpy(hd.st.dets, dets_xyxy, sizeof(float) * 4 * n_dets, cudaMemcpyHostToDevice));
    SOF_CUDA_OK(cudaMemcpy(hd.st.ndets, &n_dets, sizeof(int), cudaMemcpyHostToDevice));
    const SofDets dt{hd.st.dets, hd.st.ndets, hd.st.det_cap, 4, -1, 0.f};
    sof_enqueue(hd.st, hd.d_img, ib, rows, cols, dt, nullptr, 0);
    SOF_CUDA_OK(cudaMemcpy(warp6, hd.st.b.warp, sizeof(float) * 6, cudaMemcpyDeviceToHost));
    if (status) SOF_CUDA_OK(cudaMemcpy(status, hd.st.b.status, sizeof(int), cudaMemcpyDeviceToHost));
}

}  // namespace bmb
