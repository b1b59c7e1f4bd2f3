// reid_tc_host.cuh -- host side of the tensor-core OSNet path (included by reid_model.cu after ReidModel): weight
// packing into split-BF16 UMMA layouts, the plane workspace, tensor maps, and the per-model launch plan (every kernel
// argument, tensor map included, is built once at load; a forward pass only replays the launches).
#pragma once
#include "reid_tc.cuh"

namespace bmb {

PFN_encodeTiled tensor_map_encoder() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        RCUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        if (!p) throw std::runtime_error("cuTensorMapEncodeTiled is not available in this driver");
        fn = (PFN_encodeTiled)p;
    }
    return fn;
}

// Tensor maps over a plane tensor [crops][C8][H][W][8] of BF16.  The same bytes are described as 32-bit elements with
// long inner rows: a 16-byte inner box (one pixel of one plane) makes the TMA unit issue one request per pixel
// (3 264 per chain tile); a whole padded image row / 64 pixels per request brings that to ~100.  Out-of-bounds elements read as zero (= the convolution's zero padding).
static void encode_u32_map(CUtensorMap* out, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                           const cuuint32_t* box) {
    cuuint32_t es[5] = {1, 1, 1, 1, 1};
    CUresult r = tensor_map_encoder()(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box,
                                      es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}
// haloed row tile for the chain kernel: box = (W + 2 pixels, rows, all planes, 1 crop), start pixel -1
void make_rows_map(CUtensorMap* out, const void* base, int crops, int C8, int H, int W, int box_rows) {
    cuuint64_t dims[4] = {(cuuint64_t)W * 4, (cuuint64_t)H, (cuuint64_t)C8, (cuuint64_t)crops};
    cuuint64_t strides[3] = {(cuuint64_t)W * 16, (cuuint64_t)H * W * 16, (cuuint64_t)C8 * H * W * 16};
    cuuint32_t box[4] = {(cuuint32_t)(W + 2) * 4, (cuuint32_t)box_rows, (cuuint32_t)C8, 1};
    encode_u32_map(out, base, 4, dims, strides, box);
}
// 128 consecutive pixels of kc planes for the GEMM kernel: box = (64 pixels, 2, kc planes, 1 crop)
void make_tile_map(CUtensorMap* out, const void* base, int crops, int C8, int HW, int kc) {
    cuuint64_t dims[4] = {256, (cuuint64_t)HW / 64, (cuuint64_t)C8, (cuuint64_t)crops};
    cuuint64_t strides[3] = {1024, (cuuint64_t)HW * 16, (cuuint64_t)C8 * HW * 16};
    cuuint32_t box[4] = {256, 2, (cuuint32_t)kc, 1};
    encode_u32_map(out, base, 4, dims, strides, box);
}

namespace tcx {

inline uint16_t f2bf(float x) {   // round to nearest even, like __float2bfloat16_rn (finite inputs)
    uint32_t u;
    memcpy(&u, &x, 4);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}
inline float bf2f(uint16_t h) {
    const uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
inline int pad16(int c) { return (c + 15) / 16 * 16; }

// W[K][N] (row-major, rows >= K or columns >= N read as zero; `identity` puts 1 on the diagonal instead) ->
// [K8][2*NP][8] BF16: row n = hi of column n, row NP + n = lo.  Appends to `out`, returns the offset in elements.
inline size_t pack_b(std::vector<uint16_t>& out, const float* w, int K, int N, int ldw, int K8, int NP, int k_row0 = 0,
                     bool identity = false) {
    size_t at = out.size();
    at = (at + 63) / 64 * 64;                      // 128-byte aligned tensors
    out.resize(at + (size_t)K8 * 2 * NP * 8, 0);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) {
            const float v = identity ? (k == n ? 1.f : 0.f) : w[(size_t)k * ldw + n];
            const uint16_t h = f2bf(v);
            const int kk = k_row0 + k;
            uint16_t* plane = out.data() + at + (size_t)(kk / 8) * 2 * NP * 8;
            plane[(size_t)n * 8 + kk % 8] = h;
            plane[(size_t)(NP + n) * 8 + kk % 8] = f2bf(v - bf2f(h));
        }
    return at;
}
inline size_t pack_f(std::vector<float>& out, const float* src, int n, int n_pad) {
    size_t at = (out.size() + 3) / 4 * 4;
    out.resize(at + n_pad, 0.f);
    for (int i = 0; i < n; ++i) out[at + i] = src[i];
    return at;
}

struct Planes {
    bf16* hi = nullptr;
    bf16* lo = nullptr;
};

enum LaunchKind { LK_CHAIN_S2, LK_CHAIN_S3, LK_CHAIN_S4, LK_GEMM, LK_MAXPOOL_PLANES, LK_GATES, LK_FRONT };
struct Launch {
    int kind = LK_GEMM;
    int cls = 0;                // profiling class
    ChainTcArgs chain{};
    int chain_tiles = 0;
    GemmTcArgs gemm{};
    const bf16* src_hi[2] = {nullptr, nullptr};
    const bf16* src_lo[2] = {nullptr, nullptr};
    FrontTcArgs front{};
    GemmSmem gl{};
    GemmKernel gemm_fn = nullptr;   // the k_gemm_tc instance of (NP, NP2, epilogue mode)
    int gemm_ctas = 0;              // its CTAs per SM at layout gl, as the occupancy calculator reports them
    int gemm_groups = 0;
    int stage_after = -1;       // debug stage index whose tensor exists after this launch
    // the tensor to expose when a debug stop hits here
    const bf16* dbg_hi = nullptr;
    const bf16* dbg_lo = nullptr;
    int dbg_C8 = 0, dbg_HW = 0, dbg_C = 0;
};

struct Plan {
    int chunk = 0;
    bool head_fused = false;    // `launches` ends with conv5 + head in one kernel (`launches_dbg` keeps conv5 -> k_head)
    bf16* d_wb = nullptr;       // packed BF16 weights
    float* d_wf = nullptr;      // padded float32 side tables (bias, depthwise taps)
    Planes P, X1, Y, XA, XB;
    float* c5 = nullptr;        // conv5 output [crops][128][C3] float32
    float* sums[4] = {nullptr, nullptr, nullptr, nullptr};
    float* gates = nullptr;     // [crops][4][midp]
    int* arrivals = nullptr;    // per-crop CTA arrival counters of k_chain_tc (self-resetting)
    bf16* bfold = nullptr;      // per-crop gate-folded conv3 rows of the combine GEMM's B operand
    float* dbg_crop = nullptr;  // resized crops of the fused front kernel (diagnostics, allocated on first use)
    float* dbg = nullptr;       // float32 NHWC copy of a stage (diagnostics)
    std::vector<Launch> launches;      // product path (transition fused behind the second block of stages 2 and 3)
    std::vector<Launch> launches_dbg;  // same network, every block output materialised (diagnostic stops)
    int smem_limit = 0;
};

inline void alloc_planes(Planes& p, size_t elems) {
    RCUDA_OK(cudaMalloc(&p.hi, elems * 2));
    RCUDA_OK(cudaMalloc(&p.lo, elems * 2));
}
inline void free_planes(Planes& p) {
    cudaFree(p.hi);
    cudaFree(p.lo);
    p.hi = p.lo = nullptr;
}

inline void plan_free(Plan* p) {
    if (!p) return;
    cudaFree(p->d_wb); cudaFree(p->d_wf); cudaFree(p->c5); cudaFree(p->dbg); cudaFree(p->gates); cudaFree(p->bfold); cudaFree(p->arrivals); cudaFree(p->dbg_crop);
    for (int b = 0; b < 4; ++b) cudaFree(p->sums[b]);
    free_planes(p->P); free_planes(p->X1); free_planes(p->Y); free_planes(p->XA); free_planes(p->XB);
    delete p;
}

}  // namespace tcx
}  // namespace bmb
