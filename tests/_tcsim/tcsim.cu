// tcsim.cu -- test harness for the tensor-core OSNet kernels (tests only; never a product path).
//
// Includes the product headers unchanged and launches one k_gemm_tc instance or one k_chain_tc shape at a time, with
// the operands packed by the product's own host code (pack_b, make_tile_map, make_rows_map, gemm_smem_layout), so
// that tests/test_gpu_reid_tc_kernels.py can pin every instance, ring depth, ring chunk, tile grouping and crop window
// against a float64 reference.  The host-only entry points (f2bf / the hi-lo split, pack_b, pack_f, the instance table,
// the shared-memory layout) need no GPU; tests/test_tcsim_host.py pins the Python encoders on them.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "engine.h"

#define RCUDA_OK(expr)                                                                                  \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess)                                                                          \
            throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e));              \
    } while (0)

#include "reid_tc_host.cuh"

using namespace bmb;
using namespace bmb::tcx;

namespace {

std::string g_err;

// device allocations of one harness call, freed on every exit path
struct DevMem {
    std::vector<void*> ptrs;
    ~DevMem() {
        for (void* p : ptrs) cudaFree(p);
    }
    template <class T>
    T* alloc(size_t n) {
        void* p = nullptr;
        RCUDA_OK(cudaMalloc(&p, n * sizeof(T) + 256));
        ptrs.push_back(p);
        return static_cast<T*>(p);
    }
    template <class T>
    T* upload(const T* h, size_t n) {
        T* d = alloc<T>(n);
        RCUDA_OK(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice));
        return d;
    }
};

template <class T>
void download(T* h, const T* d, size_t n) {
    RCUDA_OK(cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost));
}

// float32 NHWC [crops][HW][C8 * 8] -> split planes [crops][C8][HW][8] (hi = f2bf(x), lo = f2bf(x - hi))
void to_planes(const float* x, int crops, int HW, int C8, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
    const size_t n = (size_t)crops * HW * C8 * 8;
    hi.assign(n, 0);
    lo.assign(n, 0);
    for (int c = 0; c < crops; ++c)
        for (int p = 0; p < HW; ++p)
            for (int k = 0; k < C8 * 8; ++k) {
                const float v = x[((size_t)c * HW + p) * C8 * 8 + k];
                const size_t o = (((size_t)c * C8 + k / 8) * HW + p) * 8 + k % 8;
                hi[o] = f2bf(v);
                lo[o] = f2bf(v - bf2f(hi[o]));
            }
}

template <int... I>
int min_ctas_of(int np, int np2, int mode, std::integer_sequence<int, I...>) {
    int r = 0;
    ((np == 16 * (I / 45 + 1) && np2 == 16 * ((I / 5) % 9) && mode == I % 5
          ? (void)(r = gemm_min_ctas<16 * (I / 45 + 1), 16 * ((I / 5) % 9), I % 5>())
          : (void)0),
     ...);
    return r;
}

int smem_limit_optin() {
    int dev = 0, lim = 0;
    RCUDA_OK(cudaGetDevice(&dev));
    RCUDA_OK(cudaDeviceGetAttribute(&lim, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    return lim - 1024;   // as plan_build: the static shared memory comes out of the same budget
}

}  // namespace

extern "C" {

const char* tcsim_last_error() { return g_err.c_str(); }

// ---- host-only ------------------------------------------------------------------------------------------------
void tcsim_f2bf(const float* x, long long n, uint16_t* out) {
    for (long long i = 0; i < n; ++i) out[i] = f2bf(x[i]);
}
// the split of pack_b: hi = f2bf(x), lo = f2bf(x - bf2f(hi))
void tcsim_split(const float* x, long long n, uint16_t* hi, uint16_t* lo) {
    for (long long i = 0; i < n; ++i) {
        hi[i] = f2bf(x[i]);
        lo[i] = f2bf(x[i] - bf2f(hi[i]));
    }
}
// pack_b appended to a vector that already holds `prefix` elements; copies the packed block ([K8][2 NP][8]) to `out`
// and returns the offset pack_b reported
long long tcsim_pack_b(const float* w, int K, int N, int ldw, int K8, int NP, int k_row0, int identity, int prefix,
                       uint16_t* out) {
    std::vector<uint16_t> v((size_t)prefix, 0x7fc1);
    const size_t at = pack_b(v, w, K, N, ldw, K8, NP, k_row0, identity != 0);
    memcpy(out, v.data() + at, (size_t)K8 * 2 * NP * 8 * sizeof(uint16_t));
    return (long long)at;
}
long long tcsim_pack_f(const float* src, int n, int n_pad, int prefix, float* out) {
    std::vector<float> v((size_t)prefix, -1.f);
    const size_t at = pack_f(v, src, n, n_pad);
    memcpy(out, v.data() + at, (size_t)n_pad * sizeof(float));
    return (long long)at;
}
int tcsim_n_instances() { return (int)(sizeof(kGemmInstances) / sizeof(kGemmInstances[0])); }
void tcsim_instance(int i, int* np, int* np2, int* mode, int* min_ctas) {
    const GemmInstance& g = kGemmInstances[i];
    *np = g.NP;
    *np2 = g.NP2;
    *mode = g.mode;
    *min_ctas = min_ctas_of(g.NP, g.NP2, g.mode, std::make_integer_sequence<int, 8 * 9 * 5>{});
}
// b, b2, ring, a2, f, gate, total
void tcsim_smem_layout(int K8, int NP, int NP2, int n_stage, int tail, int pool, int slot_bytes, int pool2, long long* out) {
    const GemmSmem s = gemm_smem_layout(K8, NP, NP2, n_stage, tail != 0, pool != 0, slot_bytes, pool2 != 0);
    const size_t v[7] = {s.b, s.b2, s.ring, s.a2, s.f, s.gate, s.total};
    for (int i = 0; i < 7; ++i) out[i] = (long long)v[i];
}

// ---- device --------------------------------------------------------------------------------------------------------
int tcsim_smem_limit() {
    try {
        return smem_limit_optin();
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
}

struct TcsimGemmCfg {
    int NP, NP2, mode;
    int H, W;
    int n_src, c8[2], kc[2];
    int n_stage, tiles_per_cta;
    int relu;
    int midp;          // > 0: the first 4 * midp rows of B come per crop from `wfold` (gate-folded conv3)
    int out_planes;    // write the output planes (out_hi / out_lo)
    int out_f32;       // write the float32 NHWC copy
    int N, N2;
    int feat, out_ld;  // head
    int cap, off, count;
};
struct TcsimGemmIO {
    const float* a[2];        // per source [cap][HW][c8 * 8] float32
    const float* w;           // [K][N] float32, K = 8 * (c8[0] + c8[1]); rows below 4 * midp are not read by the kernel
    const float* bias;        // [NP]
    const float* wfold;       // [cap][4 * midp][N]
    const float* w2;          // [NP][N2]
    const float* bias2;       // [NP2]
    const float* head_w;      // [N][feat]
    const float* head_b;      // [feat]
    const int* out_row;       // [off + cap]
    // outputs, filled with canaries by the caller and returned whole (sizes in elements)
    uint16_t* out_hi; uint16_t* out_lo; long long out_n;
    uint16_t* out2_hi; uint16_t* out2_lo; long long out2_n;
    float* out_f32; long long f32_n;
    float* head_out; long long head_n;
};

// One launch of k_gemm_tc<NP, NP2, mode>.  Returns 0 (info: smem bytes, CTAs per SM, grid x), 1 when the layout does not
// fit the opt-in shared memory, -1 on an error (tcsim_last_error).
int tcsim_gemm(const TcsimGemmCfg* cp, const TcsimGemmIO* io, int* info) {
    try {
        const TcsimGemmCfg& c = *cp;
        const GemmKernel fn = gemm_instance(c.NP, c.NP2, c.mode);
        if (!fn) throw std::runtime_error("no k_gemm_tc instance for this (NP, NP2, mode)");
        const bool tail = c.mode == GM_TAIL || c.mode == GM_TAIL_POOL2, pool = c.mode == GM_POOL, pool2 = c.mode == GM_TAIL_POOL2;
        const bool head = c.mode == GM_HEAD;
        const int HW = c.H * c.W;
        if (HW % 128) throw std::runtime_error("HW must be a multiple of 128");
        DevMem dm;
        GemmTcArgs g{};
        g.n_src = c.n_src;
        g.rows_per_tile = 128 / c.W;
        g.tiles_per_crop = HW / 128;
        g.tiles_per_cta = c.tiles_per_cta;
        g.n_stage = c.n_stage;
        g.K8 = 0;
        int kc_max = 2;
        for (int s = 0; s < c.n_src; ++s) {
            if (c.kc[s] < 2 || c.kc[s] % 2 || c.c8[s] % c.kc[s]) throw std::runtime_error("kc must be even and divide C8");
            std::vector<uint16_t> hi, lo;
            to_planes(io->a[s], c.cap, HW, c.c8[s], hi, lo);
            const bf16* dh = reinterpret_cast<const bf16*>(dm.upload(hi.data(), hi.size()));
            const bf16* dl = reinterpret_cast<const bf16*>(dm.upload(lo.data(), lo.size()));
            make_tile_map(&g.map_hi[s], dh, c.cap, c.c8[s], HW, c.kc[s]);
            make_tile_map(&g.map_lo[s], dl, c.cap, c.c8[s], HW, c.kc[s]);
            g.src_planes[s] = c.c8[s];
            g.src_kc[s] = c.kc[s];
            g.K8 += c.c8[s];
            kc_max = std::max(kc_max, c.kc[s]);
        }
        g.slot_bytes = kc_max * 128 * 16 * 2;
        const int K = g.K8 * 8;
        std::vector<uint16_t> wb;
        pack_b(wb, io->w, K, c.N, c.N, g.K8, c.NP);
        g.b_packed = reinterpret_cast<const bf16*>(dm.upload(wb.data(), wb.size()));
        g.N = c.N;
        g.NP = c.NP;
        g.bias = dm.upload(io->bias, (size_t)c.NP);
        g.relu = c.relu;
        g.HW = HW;
        g.W = c.W;
        if (c.midp > 0) {   // per-crop gate-folded rows, packed as gates_fold writes them
            const int rows = 4 * c.midp;
            std::vector<uint16_t> fold;
            for (int n = 0; n < c.cap; ++n) {
                std::vector<uint16_t> one;
                pack_b(one, io->wfold + (size_t)n * rows * c.N, rows, c.N, c.N, rows / 8, c.NP);
                fold.insert(fold.end(), one.begin(), one.end());
            }
            g.bfold = reinterpret_cast<const bf16*>(dm.upload(fold.data(), fold.size()));
            g.midp = c.midp;
        }
        if (c.out_planes) {
            g.out_hi = reinterpret_cast<bf16*>(dm.upload(io->out_hi, (size_t)io->out_n));
            g.out_lo = reinterpret_cast<bf16*>(dm.upload(io->out_lo, (size_t)io->out_n));
        }
        if (c.out_f32) g.out_f32 = dm.upload(io->out_f32, (size_t)io->f32_n);
        g.pool = pool ? 1 : 0;
        g.pool2 = pool2 ? 1 : 0;
        if (tail) {
            std::vector<uint16_t> w2;
            pack_b(w2, io->w2, c.NP, c.N2, c.N2, c.NP / 8, c.NP2);
            g.b2_packed = reinterpret_cast<const bf16*>(dm.upload(w2.data(), w2.size()));
            g.bias2 = dm.upload(io->bias2, (size_t)c.NP2);
            g.N2 = c.N2;
            g.NP2 = c.NP2;
            g.out2_hi = reinterpret_cast<bf16*>(dm.upload(io->out2_hi, (size_t)io->out2_n));
            g.out2_lo = reinterpret_cast<bf16*>(dm.upload(io->out2_lo, (size_t)io->out2_n));
        }
        GemmHeadIO hio{};
        float* d_head = nullptr;
        if (head) {
            g.head_w = dm.upload(io->head_w, (size_t)c.N * c.feat);
            g.head_b = dm.upload(io->head_b, (size_t)c.feat);
            g.head_feat = c.feat;
            std::vector<CropDesc> cd((size_t)c.off + c.cap);
            for (size_t i = 0; i < cd.size(); ++i) cd[i] = CropDesc{0.f, 0.f, 1.f, 1.f, 0, io->out_row[i]};
            hio.crops = dm.upload(cd.data(), cd.size());
            d_head = dm.upload(io->head_out, (size_t)io->head_n);
            hio.out = d_head;
            hio.out_ld = c.out_ld;
        }
        const GemmSmem L = gemm_smem_layout(g.K8, g.NP, tail ? g.NP2 : 0, g.n_stage, tail, pool, g.slot_bytes, pool2);
        const int limit = smem_limit_optin();
        if ((long long)L.total > limit) return 1;
        RCUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, limit));
        int ctas = 0;
        RCUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, fn, GEMM_THREADS, L.total));
        if (ctas < 1) return 1;
        int* d_n = dm.upload(&c.count, 1);
        const int groups = (g.tiles_per_crop + g.tiles_per_cta - 1) / g.tiles_per_cta;
        fn<<<dim3(groups, c.cap), GEMM_THREADS, L.total>>>(g, d_n, c.off, c.cap, L, hio);
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaDeviceSynchronize());
        if (c.out_planes) {
            download(io->out_hi, reinterpret_cast<uint16_t*>(g.out_hi), (size_t)io->out_n);
            download(io->out_lo, reinterpret_cast<uint16_t*>(g.out_lo), (size_t)io->out_n);
        }
        if (c.out_f32) download(io->out_f32, g.out_f32, (size_t)io->f32_n);
        if (tail) {
            download(io->out2_hi, reinterpret_cast<uint16_t*>(g.out2_hi), (size_t)io->out2_n);
            download(io->out2_lo, reinterpret_cast<uint16_t*>(g.out2_lo), (size_t)io->out2_n);
        }
        if (head) download(io->head_out, d_head, (size_t)io->head_n);
        info[0] = (int)L.total;
        info[1] = ctas;
        info[2] = groups;
        return 0;
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"

struct TcsimChainCfg {
    int shape;           // 0, 1, 2: BMB_CHAIN_S2 / S3 / S4
    int mid, hid, N;     // LightConv channels (= CR), ChannelGate hidden width, conv3 output channels
    int cap, off;
    int n_launch;        // consecutive launches on one set of buffers, launch i with count counts[i] and input x[i]
    int counts[4];
};
struct TcsimChainIO {
    const float* x;      // [n_launch][cap][H][W][CP] float32 (conv1's output; channels >= mid are zero)
    const float* pw;     // [10][mid][mid]  1x1 weights (in, out)
    const float* dw;     // [10][9][mid]    depthwise taps (BN folded), tap = ky * 3 + kx
    const float* b;      // [10][mid]
    const float* g1w; const float* g1b; const float* g2w; const float* g2b;   // [mid][hid], [hid], [hid][mid], [mid]
    const float* w3;     // [mid][N]
    // outputs, filled with canaries by the caller
    uint16_t* y_hi; uint16_t* y_lo;   // [cap][4 CP / 8][H][W][8]
    float* sums;                      // [4][cap][tiles][CP]
    float* gates;                     // [cap][4][CP]
    uint16_t* bfold;                  // [cap][4 CP / 8][2 NP][8]
    int* arrivals;                    // [cap]
};

template <int CP, int CR, int W, int R, int NSPLIT>
static int chain_run(const TcsimChainCfg& c, const TcsimChainIO& io, int H) {
    DevMem dm;
    const int C8 = CP / 8, HW = H * W, tiles = H / R, NP = pad16(c.N);
    if (c.mid != CR) throw std::runtime_error("mid does not match the chain shape");
    std::vector<uint16_t> wb;
    size_t pw_at[10];
    for (int l = 0; l < 10; ++l) pw_at[l] = pack_b(wb, io.pw + (size_t)l * CR * CR, CR, CR, CR, C8, CP);
    const bf16* d_wb = reinterpret_cast<const bf16*>(dm.upload(wb.data(), wb.size()));
    std::vector<float> wf;
    size_t dw_at[10];
    for (int l = 0; l < 10; ++l) {   // taps [9][CP] and the bias right behind them (one bulk copy), as plan_build lays them out
        size_t at = (wf.size() + 31) / 32 * 32;
        wf.resize(at + 10 * CP, 0.f);
        for (int t = 0; t < 9; ++t)
            for (int ch = 0; ch < CR; ++ch) wf[at + t * CP + ch] = io.dw[((size_t)l * 9 + t) * CR + ch];
        for (int ch = 0; ch < CR; ++ch) wf[at + 9 * CP + ch] = io.b[(size_t)l * CR + ch];
        dw_at[l] = at;
    }
    const float* d_wf = dm.upload(wf.data(), wf.size());
    ChainTcArgs a{};
    for (int l = 0; l < 10; ++l) {
        a.wpw[l] = d_wb + pw_at[l];
        a.wdw[l] = d_wf + dw_at[l];
        a.bias[l] = d_wf + dw_at[l] + 9 * CP;
    }
    const size_t y_n = (size_t)c.cap * 4 * C8 * HW * 8, s_n = (size_t)c.cap * tiles * CP;
    a.y_hi = reinterpret_cast<bf16*>(dm.upload(io.y_hi, y_n));
    a.y_lo = reinterpret_cast<bf16*>(dm.upload(io.y_lo, y_n));
    float* d_sums = dm.upload(io.sums, 4 * s_n);
    for (int b = 0; b < 4; ++b) a.sums[b] = d_sums + b * s_n;
    a.H = H;
    GatesTcArgs& ga = a.gate;
    for (int b = 0; b < 4; ++b) ga.sums[b] = a.sums[b];
    ga.g1w = dm.upload(io.g1w, (size_t)CR * c.hid);
    ga.g1b = dm.upload(io.g1b, (size_t)c.hid);
    ga.g2w = dm.upload(io.g2w, (size_t)c.hid * CR);
    ga.g2b = dm.upload(io.g2b, (size_t)CR);
    ga.gates = dm.upload(io.gates, (size_t)c.cap * 4 * CP);
    ga.mid = CR;
    ga.midp = CP;
    ga.hid = c.hid;
    ga.tiles = tiles;
    ga.HW = HW;
    ga.w3 = dm.upload(io.w3, (size_t)CR * c.N);
    const size_t fold_n = (size_t)c.cap * (4 * CP / 8) * 2 * NP * 8;
    ga.bfold = reinterpret_cast<bf16*>(dm.upload(io.bfold, fold_n));
    ga.N = c.N;
    ga.NP = NP;
    ga.arrivals = dm.alloc<int>((size_t)c.cap);
    RCUDA_OK(cudaMemset(ga.arrivals, 0, sizeof(int) * c.cap));
    RCUDA_OK((chain_prepare<CP, CR, W, R, NSPLIT>()));
    int* d_n = dm.alloc<int>(1);
    const size_t x_n = (size_t)c.cap * HW * CP;
    bf16* d_xh = reinterpret_cast<bf16*>(dm.alloc<uint16_t>(x_n));
    bf16* d_xl = reinterpret_cast<bf16*>(dm.alloc<uint16_t>(x_n));
    make_rows_map(&a.map_hi, d_xh, c.cap, C8, H, W, R + 8);
    make_rows_map(&a.map_lo, d_xl, c.cap, C8, H, W, R + 8);
    for (int i = 0; i < c.n_launch; ++i) {
        std::vector<uint16_t> hi, lo;
        to_planes(io.x + (size_t)i * x_n, c.cap, HW, C8, hi, lo);
        RCUDA_OK(cudaMemcpy(d_xh, hi.data(), x_n * 2, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(d_xl, lo.data(), x_n * 2, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMemcpy(d_n, &c.counts[i], sizeof(int), cudaMemcpyHostToDevice));
        chain_launch<CP, CR, W, R, NSPLIT>(a, tiles, c.cap, d_n, c.off, 0);
        RCUDA_OK(cudaGetLastError());
        RCUDA_OK(cudaDeviceSynchronize());
    }
    download(io.y_hi, reinterpret_cast<uint16_t*>(a.y_hi), y_n);
    download(io.y_lo, reinterpret_cast<uint16_t*>(a.y_lo), y_n);
    download(io.sums, d_sums, 4 * s_n);
    download(io.gates, ga.gates, (size_t)c.cap * 4 * CP);
    download(io.bfold, reinterpret_cast<uint16_t*>(ga.bfold), fold_n);
    download(io.arrivals, ga.arrivals, (size_t)c.cap);
    return 0;
}

template <int CP, int CR, int W, int R, int NSPLIT>
static void chain_geom(int H, int* out5) {
    out5[0] = CP; out5[1] = CR; out5[2] = W; out5[3] = H; out5[4] = R;
}

extern "C" {

// geometry of a chain shape: CP, CR, W, H, R
void tcsim_chain_shape(int shape, int* out5) {
    if (shape == 0) chain_geom<BMB_CHAIN_S2>(64, out5);
    else if (shape == 1) chain_geom<BMB_CHAIN_S3>(32, out5);
    else chain_geom<BMB_CHAIN_S4>(16, out5);
}

int tcsim_chain(const TcsimChainCfg* cp, const TcsimChainIO* io) {
    try {
        switch (cp->shape) {
            case 0: return chain_run<BMB_CHAIN_S2>(*cp, *io, 64);
            case 1: return chain_run<BMB_CHAIN_S3>(*cp, *io, 32);
            case 2: return chain_run<BMB_CHAIN_S4>(*cp, *io, 16);
        }
        throw std::runtime_error("chain shape must be 0, 1 or 2");
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
}

}  // extern "C"
