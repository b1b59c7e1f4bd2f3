// reid_tc.cuh -- the tensor-core OSNet path for Hopper: every 1x1 convolution of the network runs as wgmma (BF16 split
// operands read from shared memory, FP32 accumulators in registers), activations travel between kernels as
// channel-blocked BF16 "hi + lo" planes that TMA boxes (cp.async.bulk.tensor, zero fill = convolution padding) drop
// straight into the canonical no-swizzle K-major operand layout, the depthwise 3x3 / bias / ReLU / gate / pooling
// epilogues run on the CUDA cores between the MMAs.
//
// Replaces (relative to boxmot):  reid/backbones/osnet.py:63-155 (Conv1x1, Conv1x1Linear, LightConv3x3), :161-210
// (ChannelGate), :212-260 (OSBlock), :380-405 (featuremaps after the stem) in eval mode.
//
// Numerics: a float32 value x is carried as hi = bf16(x), lo = bf16(x - hi) (|x - hi - lo| <= 2^-17 |x|); a product
// A*W is evaluated as  A_hi*W_hi + A_lo*W_hi + A_hi*W_lo  with FP32 accumulation (the dropped lo*lo term is 2^-16
// relative).  Where the weights are stored as [W_hi | W_lo] along the output channel, A_hi x [W_hi | W_lo] is one
// wgmma of 2N columns and A_lo x W_hi accumulates into its first N columns; the epilogue adds the two column groups.
//
// Kernels:
//   k_chain_tc   one OSBlock branch (1-4 LightConv3x3 = 1x1 -> depthwise 3x3 -> BN -> ReLU) per CTA on a haloed row
//                tile: TMA box of conv1's output -> [wgmma 1x1 -> T (smem, fp32) -> depthwise on CUDA cores -> split
//                planes in place] x depth -> branch output planes + channel sums for the gate.
//   k_gemm_tc    warp-specialised pointwise GEMM (TMA producer warp / two consumer warpgroups, 64 pixels each) over
//                128-pixel tiles, one instance per output width and epilogue mode: A = up to two plane tensors streamed
//                through an mbarrier ring (MMAs pipelined one k-step deep), B resident in shared
//                memory (optionally  gate (x) conv3  folded per crop), epilogue bias + ReLU -> planes, optional 2x2
//                average pool, optional float32 NHWC copy, optional second GEMM on the fresh tile (next block's conv1).
#pragma once
#include "wgmma.cuh"

namespace bmb {
namespace tcx {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ int tc_chunk_count(const int* d_n, int off, int cap) {
    int n = *d_n - off;
    n = n < 0 ? 0 : n;
    return n > cap ? cap : n;
}
using um::mbar_arrive;

// ------------------------------------------------------------------------------------------------------------------
// maxpool 3x3 stride 2 pad 1 on the stem output (float32 NHWC) -> split planes  [crops][C/8][H/2][W/2][8]
// ------------------------------------------------------------------------------------------------------------------
__global__ void k_maxpool_planes(const float* __restrict__ in, int H, int W, int C, const int* __restrict__ d_n, int off,
                                 int cap, bf16* __restrict__ out_hi, bf16* __restrict__ out_lo) {
    const int n_crops = tc_chunk_count(d_n, off, cap);
    const int OH = H / 2, OW = W / 2, C8 = C / 8;
    const size_t total = (size_t)n_crops * C8 * OH * OW;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int ox = (int)(e % OW);
        size_t r = e / OW;
        const int oy = (int)(r % OH); r /= OH;
        const int c8 = (int)(r % C8);
        const int n = (int)(r / C8);
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * 2 - 1 + ky;
            if (iy < 0 || iy >= H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * 2 - 1 + kx;
                if (ix < 0 || ix >= W) continue;
                const float4* p = reinterpret_cast<const float4*>(in + (((size_t)n * H + iy) * W + ix) * C + c8 * 8);
                const float4 a = p[0], b = p[1];
                m[0] = fmaxf(m[0], a.x); m[1] = fmaxf(m[1], a.y); m[2] = fmaxf(m[2], a.z); m[3] = fmaxf(m[3], a.w);
                m[4] = fmaxf(m[4], b.x); m[5] = fmaxf(m[5], b.y); m[6] = fmaxf(m[6], b.z); m[7] = fmaxf(m[7], b.w);
            }
        }
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) um::split2(m[2 * j], m[2 * j + 1], h[j], l[j]);
        reinterpret_cast<uint4*>(out_hi)[e] = make_uint4(h[0], h[1], h[2], h[3]);
        reinterpret_cast<uint4*>(out_lo)[e] = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

// planes -> float32 NHWC (diagnostics: the per-stage parity test reads block outputs through this)
__global__ void k_planes_to_nhwc(const bf16* __restrict__ hi, const bf16* __restrict__ lo, int C8, int HW, int C_real,
                                 const int* __restrict__ d_n, int off, int cap, float* __restrict__ out) {
    const int n_crops = tc_chunk_count(d_n, off, cap);
    const size_t total = (size_t)n_crops * C8 * HW;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const int p = (int)(e % HW);
        size_t r = e / HW;
        const int c8 = (int)(r % C8);
        const int n = (int)(r / C8);
        const uint4 h = reinterpret_cast<const uint4*>(hi)[e], l = reinterpret_cast<const uint4*>(lo)[e];
        const uint32_t hh[4] = {h.x, h.y, h.z, h.w}, ll[4] = {l.x, l.y, l.z, l.w};
        float* o = out + ((size_t)n * HW + p) * C_real + c8 * 8;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 v = um::join2(hh[j], ll[j]);
            if (c8 * 8 + 2 * j < C_real) o[2 * j] = v.x;
            if (c8 * 8 + 2 * j + 1 < C_real) o[2 * j + 1] = v.y;
        }
    }
}

// ChannelGate (osnet.py:161-210) of the four branches of a block: mean -> fc1 -> ReLU -> fc2 -> sigmoid, and conv3 with
// the gates folded in (the first 4 * midp rows of the combine GEMM's B operand, per crop).  Runs in the LAST k_chain_tc
// CTA of a crop to finish (a per-crop arrival counter): no launch of its own, no redundant work.  Same operation order as
// the float32 k_gates of round 1.
struct GatesTcArgs {
    const float* sums[4];               // [crops][tiles][midp]
    const float* g1w; const float* g1b; const float* g2w; const float* g2b;   // [mid][hid], [hid], [hid][mid], [mid]
    float* gates;                       // [crops][4][midp] (padded channels 0)
    int mid, midp, hid, tiles, HW;
    // bfold[crop] = [4 * midp / 8][2 * NP][8] BF16 ([hi | lo] along n), row (b * midp + c) = gates[b][c] * w3[c][:]
    const float* w3;                    // [mid][N] float32
    bf16* bfold;
    int N, NP;
    int* arrivals;                      // [crops] CTAs of the crop that have published their channel sums
};
template <int NT>
__device__ void gates_fold(const GatesTcArgs& a, const int n, float* mean /*128*/, float* hid /*16*/, float* gate /*128*/) {
    const int mid = a.mid, midp = a.midp;
    for (int e = threadIdx.x; e < 4 * midp; e += NT) {
        const int b = e / midp, c = e - b * midp;
        float s = 0.f;
        if (c < mid)
            for (int t = 0; t < a.tiles; ++t) s += __ldcg(a.sums[b] + ((size_t)n * a.tiles + t) * midp + c);
        mean[e] = s / (float)a.HW;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 4 * a.hid; e += NT) {
        const int b = e / a.hid, h = e - b * a.hid;
        float s = a.g1b[h];
        for (int c = 0; c < mid; ++c) s = fmaf(mean[b * midp + c], a.g1w[(size_t)c * a.hid + h], s);
        hid[e] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 4 * midp; e += NT) {
        const int b = e / midp, c = e - b * midp;
        float g = 0.f;
        if (c < mid) {
            float s = a.g2b[c];
            for (int h = 0; h < a.hid; ++h) s = fmaf(hid[b * a.hid + h], a.g2w[(size_t)h * mid + c], s);
            g = 1.0f / (1.0f + expf(-s));
        }
        a.gates[(size_t)n * 4 * midp + e] = g;
        gate[e] = g;
    }
    __syncthreads();
    // an item = (plane of 8 rows k, pair of output channels): 8 k values x 2 n, written as four 16-byte rows
    const int NP = a.NP, N = a.N;
    const int items = (4 * midp / 8) * (NP / 2);
    unsigned char* dst = reinterpret_cast<unsigned char*>(a.bfold) + (size_t)n * (4 * midp / 8) * 2 * NP * 16;
    for (int e = threadIdx.x; e < items; e += NT) {
        const int k8 = e / (NP / 2), n2 = (e - k8 * (NP / 2)) * 2;
        uint32_t h0[4], l0[4], h1[4], l1[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v00 = 0.f, v01 = 0.f, v10 = 0.f, v11 = 0.f;   // (k, n), (k+1, n), (k, n+1), (k+1, n+1)
            const int k = k8 * 8 + 2 * j;
            const int b = k / midp, c = k - b * midp;            // midp is even: k and k+1 share the branch
            if (c < mid && n2 < N) {
                v00 = gate[k] * a.w3[(size_t)c * N + n2];
                if (n2 + 1 < N) v10 = gate[k] * a.w3[(size_t)c * N + n2 + 1];
            }
            if (c + 1 < mid && n2 < N) {
                v01 = gate[k + 1] * a.w3[(size_t)(c + 1) * N + n2];
                if (n2 + 1 < N) v11 = gate[k + 1] * a.w3[(size_t)(c + 1) * N + n2 + 1];
            }
            um::split2(v00, v01, h0[j], l0[j]);
            um::split2(v10, v11, h1[j], l1[j]);
        }
        unsigned char* row = dst + ((size_t)k8 * 2 * NP) * 16;
        *reinterpret_cast<uint4*>(row + (size_t)n2 * 16) = make_uint4(h0[0], h0[1], h0[2], h0[3]);
        *reinterpret_cast<uint4*>(row + (size_t)(n2 + 1) * 16) = make_uint4(h1[0], h1[1], h1[2], h1[3]);
        *reinterpret_cast<uint4*>(row + (size_t)(NP + n2) * 16) = make_uint4(l0[0], l0[1], l0[2], l0[3]);
        *reinterpret_cast<uint4*>(row + (size_t)(NP + n2 + 1) * 16) = make_uint4(l1[0], l1[1], l1[2], l1[3]);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// k_chain_tc: one branch of an OSBlock per CTA.  grid = (row tiles, 4 branches (deepest first), crops), 256 threads.
// Shared memory: X hi / lo planes [CP/8][NPX][8] (NPX = (R + 8) padded rows of W + 2 pixels; the TMA box of conv1's
// output lands here with zero fill outside the image = every layer's zero padding), T [CP/4][NPXT] float4 (1x1 result),
// two weight slots.  Per level: each warpgroup takes every other 64-pixel slice of the rows the level reads, runs two
// wgmma chains per slice (A_hi x [W_hi | W_lo], A_lo x W_hi) and adds the column groups into T, then column walkers (3x3 register window, as in the float32 kernels of round 1) apply the
// depthwise taps + bias + ReLU and write the next level's X as hi / lo planes in place; the last level goes to the
// branch-output planes in HBM and leaves per-tile channel sums for the ChannelGate.
// ------------------------------------------------------------------------------------------------------------------
struct ChainTcArgs {
    CUtensorMap map_hi, map_lo;      // conv1 output planes, box (W + 2 pixels, R + 8 rows, CP / 8 planes, 1 crop)
    const bf16* wpw[10];             // per LightConv: [CP/8][2*CP][8]  ([W_hi | W_lo] along the output channel)
    const float* wdw[10];            // [9][CP]   (BN folded)
    const float* bias[10];           // [CP]
    bf16* y_hi;                      // branch outputs [crops][4*CP/8][H][W][8]
    bf16* y_lo;
    float* sums[4];                  // [crops][tiles][CP]
    int H;
    GatesTcArgs gate;                // ChannelGate + conv3 fold, done by the crop's last CTA
};

template <int CP, int CR, int W, int R>
struct ChainGeom {
    static constexpr int TW = W + 2, ROWS = R + 8, NPX = ROWS * TW;
    static constexpr int NT_MAX = (NPX + 127) / 128;
    static constexpr int NPXT = ((NPX + 7) / 8) * 8 + 2;
    static constexpr int X_BYTES = (CP / 8) * NPX * 16;               // one of hi / lo
    static constexpr int T_BYTES = (CR / 4) * NPXT * 16;               // only the real channels pass through T
    static constexpr int WSLOT_BYTES = (CP / 8) * 2 * CP * 16 + 9 * CP * 4 + CP * 4;
    // the slices of a level end on a 128-pixel boundary, up to 127 pixels past the planes: hi runs into lo (not written
    // while MMAs run), lo into a slack of 128 pixels, so no MMA reads shared memory that another warpgroup writes
    static constexpr int X_SLACK = 128 * 16;
    static constexpr size_t SMEM = 2 * (size_t)X_BYTES + X_SLACK + T_BYTES + 2 * WSLOT_BYTES + 128;
};

template <int CP, int CR, int W, int R, int NSPLIT>
__global__ void __launch_bounds__(256) k_chain_tc(const __grid_constant__ ChainTcArgs a, const int* __restrict__ d_n, int off, int cap) {
    using G = ChainGeom<CP, CR, W, R>;
    const int n = blockIdx.z;
    if (n >= tc_chunk_count(d_n, off, cap)) return;
    const int br = 3 - (int)blockIdx.y, depth = br + 1, tile = blockIdx.x;
    const int l0 = br * (br + 1) / 2;
    const int H = a.H;
    constexpr int TW = G::TW, NPX = G::NPX, NPXT = G::NPXT, C8 = CP / 8, C4 = CR / 4, KS = CP / 16;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_tma, bar_w[2];
    unsigned char* sXh = smem;
    unsigned char* sXl = sXh + G::X_BYTES;
    float4* sT = reinterpret_cast<float4*>(sXl + G::X_BYTES + G::X_SLACK);
    unsigned char* sWs = reinterpret_cast<unsigned char*>(sT) + G::T_BYTES;
    float* sP = reinterpret_cast<float*>(sT);                     // [256 / C4][CR] channel-sum slots (after the last level)
    const int lane = threadIdx.x & 31;
    const int y0 = tile * R, g0 = y0 - 4;
#ifdef BMB_TC_CLOCKS
    long long ck[24];
    int nck = 0;
#define TCK() do { if (threadIdx.x == 0 && nck < 24) ck[nck++] = clock64(); } while (0)
#else
#define TCK() do { } while (0)
#endif
    TCK();

    // weights of level lv (1-based) -> slot (lv & 1): two bulk copies by thread 0 (the packed [W_hi | W_lo] block, and the
    // depthwise taps + bias, which the plan stores back to back), completing on the slot's barrier.  The copy for level
    // lv + 1 is issued while level lv's MMAs run; nobody waits on global memory (plain loads by all threads would stall
    // every level).
    constexpr uint32_t PW_BYTES = C8 * 2 * CP * 16, DW_BYTES = 10 * CP * 4;
    auto fetch_weights = [&](int lv) {
        unsigned char* dst = sWs + (size_t)(lv & 1) * G::WSLOT_BYTES;
        um::mbar_expect_tx(&bar_w[lv & 1], PW_BYTES + DW_BYTES);
        um::bulk_g2s(dst, a.wpw[l0 + lv - 1], PW_BYTES, &bar_w[lv & 1]);
        um::bulk_g2s(dst + PW_BYTES, a.wdw[l0 + lv - 1], DW_BYTES, &bar_w[lv & 1]);
    };

    // the input box first (its latency overlaps the weight staging): thread 0 initialises the barriers, publishes them
    // to the async proxy and issues the two TMA loads by itself
    if (threadIdx.x == 0) {
        um::mbar_init(&bar_tma, 1);
        um::mbar_init(&bar_w[0], 1);
        um::mbar_init(&bar_w[1], 1);
        um::fence_mbar_init();
        um::mbar_expect_tx(&bar_tma, 2u * G::X_BYTES);
        um::tma_load_4d(sXh, &a.map_hi, -4, g0, 0, n, &bar_tma);
        um::tma_load_4d(sXl, &a.map_lo, -4, g0, 0, n, &bar_tma);
        fetch_weights(1);
    }
    __syncthreads();
    TCK();
    um::mbar_wait(&bar_tma, 0);
    TCK();

    constexpr int walkers = W * C4;
    constexpr int n_grp = 256 / C4;
    constexpr int act = n_grp * C4;
    // row splits per walker column: as many as there are threads (NSPLIT = 0), or fewer, longer walks -- a walker's
    // 9 tap vectors and its first two window rows are a fixed cost per walk
    constexpr int n_split_max = (act / walkers) < 1 ? 1 : (act / walkers);
    constexpr int n_split = NSPLIT > 0 && NSPLIT < n_split_max ? NSPLIT : n_split_max;
    float4 psum = make_float4(0.f, 0.f, 0.f, 0.f);

    for (int lv = 1; lv <= depth; ++lv) {
        const int ext = depth - lv;
        const unsigned char* wslot = sWs + (size_t)(lv & 1) * G::WSLOT_BYTES;
        const int la = 4 - ext, lb = 4 + R + ext;              // local rows the depthwise stage produces
        const int pa = (la - 1) * TW, pb = (lb + 1) * TW;      // pixels whose 1x1 result it reads
        const int t0 = pa >> 7, t1 = (pb + 127) >> 7;
        um::mbar_wait(&bar_w[lv & 1], (uint32_t)((lv - 1) >> 1) & 1u);     // this level's weights (k-th use of the slot)
        // the other slot was last read by level lv - 1 (its MMAs were waited for, its walkers passed the barrier)
        if (threadIdx.x == 0 && lv < depth) fetch_weights(lv + 1);
        TCK();
        {   // ---- 1x1 on the tensor cores, T = (A_hi W_hi + A_lo W_hi) + A_hi W_lo, one 64-pixel slice at a time ----
            const uint32_t lbo_a = (uint32_t)NPX * 16u, lbo_b = 2u * CP * 16u;
            const uint32_t xh = um::smem_u32(sXh), xl = um::smem_u32(sXl), wb = um::smem_u32(wslot);
            const int wg = threadIdx.x >> 7, row = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
            float* sTf = reinterpret_cast<float*>(sT);
            for (int u = 2 * t0 + wg; u < 2 * t1; u += 2) {
                float acc[CP];
                um::wg_fence();
#pragma unroll
                for (int ks = 0; ks < KS; ++ks)
                    um::mma<2 * CP, false>(acc, um::make_desc(xh + (uint32_t)u * 1024u + ks * 2 * lbo_a, lbo_a, 128), wb + ks * 2 * lbo_b,
                                           lbo_b, 128, ks > 0);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks)
                    um::mma<CP, false>(acc, um::make_desc(xl + (uint32_t)u * 1024u + ks * 2 * lbo_a, lbo_a, 128), wb + ks * 2 * lbo_b,
                                       lbo_b, 128, 1);
                um::wg_commit();
                um::wg_wait_all();
                um::wg_fence_acc<CP>(acc);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int p = u * 64 + row + 8 * h;
                    if (p < NPX) {
#pragma unroll
                        for (int i = 0; i < CP / 8; ++i) {
                            const int c = 8 * i + cq;
                            if (c / 4 < C4)
                                *reinterpret_cast<float2*>(sTf + ((size_t)(c >> 2) * NPXT + p) * 4 + (c & 3)) =
                                    um::fadd2(make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]),
                                              make_float2(acc[CP / 2 + 4 * i + 2 * h], acc[CP / 2 + 4 * i + 2 * h + 1]));
                        }
                    }
                }
            }
        }
        __syncthreads();
        TCK();
        // ---- depthwise 3x3 + bias + ReLU on image rows [ya, yb): next level's X (planes, in place) or the branch output ----
        const bool last = lv == depth;
        const int ya = max(y0 - ext, 0), yb = min(y0 + R + ext, H);
        const int rows_lv = yb - ya;
        const int rows_per = (rows_lv + n_split - 1) / n_split;
        const float* sD = reinterpret_cast<const float*>(wslot + C8 * 2 * CP * 16);
        const float* sB = sD + 9 * CP;
        if (threadIdx.x < act) {
            for (int wk = threadIdx.x; wk < walkers * n_split; wk += act) {
                const int c4 = wk % C4, x = (wk / C4) % W, sp = wk / walkers;
                const int ra = ya + sp * rows_per, rb = min(ra + rows_per, yb);
                if (ra >= rb) continue;
                // channel pairs: two independent IEEE chains per pair, never contracted
                float2 wv[9][2];
#pragma unroll
                for (int t = 0; t < 9; ++t) {
                    const float4 w4 = *reinterpret_cast<const float4*>(sD + t * CP + c4 * 4);
                    wv[t][0] = make_float2(w4.x, w4.y);
                    wv[t][1] = make_float2(w4.z, w4.w);
                }
                const float4 bv4 = *reinterpret_cast<const float4*>(sB + c4 * 4);
                const float2 bv0 = make_float2(bv4.x, bv4.y), bv1 = make_float2(bv4.z, bv4.w);
                const float4* tp = sT + c4 * NPXT + (ra - 1 - g0) * TW + x;      // row ra - 1, column x - 1 of the padded row
                float2 win[3][3][2];
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4 q0 = tp[kx], q1 = tp[TW + kx];
                    win[0][kx][0] = make_float2(q0.x, q0.y); win[0][kx][1] = make_float2(q0.z, q0.w);
                    win[1][kx][0] = make_float2(q1.x, q1.y); win[1][kx][1] = make_float2(q1.z, q1.w);
                }
                tp += 2 * TW;                                                      // next row to load: ra + 1
                unsigned char* xh = sXh + ((c4 >> 1) * NPX + (ra - g0) * TW + x + 1) * 16 + (c4 & 1) * 8;
                unsigned char* xl = sXl + ((c4 >> 1) * NPX + (ra - g0) * TW + x + 1) * 16 + (c4 & 1) * 8;
                size_t go = ((((size_t)n * (4 * C8) + br * C8 + (c4 >> 1)) * H + ra) * W + x) * 8 + (c4 & 1) * 4;
                float2 ps0 = make_float2(0.f, 0.f), ps1 = make_float2(0.f, 0.f);
#ifdef BMB_DW_SPLIT_RN
#define BMB_DW_SPLIT um::split2
#else
#define BMB_DW_SPLIT um::split2_tz
#endif
#define BMB_DW_ROW(U)                                                                                                  \
                {                                                                                                      \
                    constexpr int i0 = (U) % 3, i1 = ((U) + 1) % 3, i2 = ((U) + 2) % 3;                                \
                    _Pragma("unroll") for (int kx = 0; kx < 3; ++kx) {                                                 \
                        const float4 qq = tp[kx];                                                                      \
                        win[i2][kx][0] = make_float2(qq.x, qq.y);                                                      \
                        win[i2][kx][1] = make_float2(qq.z, qq.w);                                                      \
                    }                                                                                                  \
                    tp += TW;                                                                                          \
                    /* three independent partial sums per channel pair (one per window row): 6 chains of 3 FFMA2 */   \
                    float2 a0 = bv0, a1 = bv1;                                                                         \
                    float2 b0 = um::fmul2(win[i1][0][0], wv[3][0]), b1 = um::fmul2(win[i1][0][1], wv[3][1]);          \
                    float2 c0 = um::fmul2(win[i2][0][0], wv[6][0]), c1 = um::fmul2(win[i2][0][1], wv[6][1]);          \
                    a0 = um::ffma2(win[i0][0][0], wv[0][0], a0);                                                      \
                    a1 = um::ffma2(win[i0][0][1], wv[0][1], a1);                                                      \
                    _Pragma("unroll") for (int kx = 1; kx < 3; ++kx) {                                                 \
                        a0 = um::ffma2(win[i0][kx][0], wv[kx][0], a0);                                                \
                        a1 = um::ffma2(win[i0][kx][1], wv[kx][1], a1);                                                \
                        b0 = um::ffma2(win[i1][kx][0], wv[3 + kx][0], b0);                                            \
                        b1 = um::ffma2(win[i1][kx][1], wv[3 + kx][1], b1);                                            \
                        c0 = um::ffma2(win[i2][kx][0], wv[6 + kx][0], c0);                                            \
                        c1 = um::ffma2(win[i2][kx][1], wv[6 + kx][1], c1);                                            \
                    }                                                                                                  \
                    a0 = um::fadd2(um::fadd2(a0, b0), c0);                                                           \
                    a1 = um::fadd2(um::fadd2(a1, b1), c1);                                                           \
                    a0.x = fmaxf(a0.x, 0.f); a0.y = fmaxf(a0.y, 0.f);                                                  \
                    a1.x = fmaxf(a1.x, 0.f); a1.y = fmaxf(a1.y, 0.f);                                                  \
                    uint32_t h0, h1, e0, e1;                                                                           \
                    BMB_DW_SPLIT(a0.x, a0.y, h0, e0);                                                                  \
                    BMB_DW_SPLIT(a1.x, a1.y, h1, e1);                                                                  \
                    if (last) {                                                                                        \
                        *reinterpret_cast<uint2*>(a.y_hi + go) = make_uint2(h0, h1);                                   \
                        *reinterpret_cast<uint2*>(a.y_lo + go) = make_uint2(e0, e1);                                   \
                        go += (size_t)W * 8;                                                                           \
                        ps0 = um::fadd2(ps0, a0);                                                                     \
                        ps1 = um::fadd2(ps1, a1);                                                                     \
                    } else {                                                                                           \
                        *reinterpret_cast<uint2*>(xh) = make_uint2(h0, h1);                                            \
                        *reinterpret_cast<uint2*>(xl) = make_uint2(e0, e1);                                            \
                        xh += TW * 16;                                                                                 \
                        xl += TW * 16;                                                                                 \
                    }                                                                                                  \
                }
                int y = ra;
                for (; y + 3 <= rb; y += 3) {
                    BMB_DW_ROW(0)
                    BMB_DW_ROW(1)
                    BMB_DW_ROW(2)
                }
                if (y < rb) BMB_DW_ROW(0)
                if (y + 1 < rb) BMB_DW_ROW(1)
#undef BMB_DW_ROW
                psum.x += ps0.x; psum.y += ps0.y; psum.z += ps1.x; psum.w += ps1.y;
            }
        }
        if (last && CP > CR) {
            // padded channels of the branch output are defined zeros (the gate-folded conv3 rows they meet are zero,
            // but stale bits could be NaN patterns)
            constexpr int PP = (CP - CR) / 8;
            static_assert((CP - CR) % 8 == 0, "channel padding must be whole planes");
            for (int e = threadIdx.x; e < PP * rows_lv * W; e += 256) {
                const int pl = e / (rows_lv * W), r = e - pl * (rows_lv * W);
                const size_t o = (((size_t)n * (4 * C8) + br * C8 + CR / 8 + pl) * H + ya) * W + r;
                reinterpret_cast<uint4*>(a.y_hi)[o] = make_uint4(0u, 0u, 0u, 0u);
                reinterpret_cast<uint4*>(a.y_lo)[o] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        um::fence_async_smem();
        __syncthreads();
        TCK();
    }
#ifdef BMB_TC_CLOCKS
    if (threadIdx.x == 0 && blockIdx.x == 1 && n == 5) {
        printf("chain CP%d W%d br%d: setup %lld tma %lld |", CP, W, br, ck[1] - ck[0], ck[2] - ck[1]);
        for (int i = 2; i + 3 < nck + 1 && i + 3 <= 23; i += 3)
            printf(" wait %lld mma %lld dw %lld |", ck[i + 1] - ck[i], ck[i + 2] - ck[i + 1], ck[i + 3] - ck[i + 2]);
        printf(" total %lld\n", ck[nck - 1] - ck[0]);
    }
#endif
    // per-tile channel sums of the branch output (fixed slot per thread, fixed combination order)
    if (threadIdx.x < act)
        *reinterpret_cast<float4*>(sP + (threadIdx.x / C4) * CR + (threadIdx.x % C4) * 4) = psum;
    __syncthreads();
    for (int c = threadIdx.x; c < CP; c += 256) {
        float s = 0.f;
        if (c < CR)
            for (int g = 0; g < n_grp; ++g) s += sP[g * CR + c];
        a.sums[br][((size_t)n * gridDim.x + tile) * CP + c] = s;
    }
    __threadfence();                                   // publish the sums before counting this CTA in
    __syncthreads();
    // the last CTA of the crop (tiles x 4 branches) turns the sums into gates and folds them into conv3
    __shared__ int s_last;
    __shared__ float s_mean[128], s_hid[16], s_gate[128];
    if (threadIdx.x == 0) {
        const int total = (int)gridDim.x * 4;
        const int prev = atomicAdd(a.gate.arrivals + n, 1);
        s_last = prev == total - 1;
        if (s_last) a.gate.arrivals[n] = 0;            // ready for the next block's launch
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        gates_fold<256>(a.gate, n, s_mean, s_hid, s_gate);
    }
}

// the three instances of OSNet_x0_25 (<CP, CR, W, R, NSPLIT>): stage 2 = 16 channels on 64 x 32, stage 3 = 24 (padded to 32)
// on 32 x 16, stage 4 = 32 on 16 x 8
// (tuning knobs for scripts/variant_build.sh: -DBMB_S3_R=8 ...)
#ifndef BMB_S2_NS
#define BMB_S2_NS 0
#endif
#ifndef BMB_S3_R
#define BMB_S3_R 16
#endif
#ifndef BMB_S3_NS
#define BMB_S3_NS 0
#endif
#ifndef BMB_S4_NS
#define BMB_S4_NS 0
#endif
#define BMB_CHAIN_S2 16, 16, 32, 16, BMB_S2_NS
#define BMB_CHAIN_S3 32, 24, 16, BMB_S3_R, BMB_S3_NS
#define BMB_CHAIN_S4 32, 32, 8, 16, BMB_S4_NS
template <int CP, int CR, int W, int R, int NSPLIT>
inline cudaError_t chain_prepare() {
    return cudaFuncSetAttribute(k_chain_tc<CP, CR, W, R, NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ChainGeom<CP, CR, W, R>::SMEM);
}
template <int CP, int CR, int W, int R, int NSPLIT>
inline void chain_launch(const ChainTcArgs& a, int tiles, int crops, const int* d_n, int off, cudaStream_t st) {
    k_chain_tc<CP, CR, W, R, NSPLIT><<<dim3(tiles, 4, crops), 256, ChainGeom<CP, CR, W, R>::SMEM, st>>>(a, d_n, off, crops);
}
template <int CP, int CR, int W, int R, int NSPLIT>
constexpr int chain_rows() { return R; }

// ------------------------------------------------------------------------------------------------------------------
// k_gemm_tc: out[p][n] = act( sum_src sum_k A_src[p][k] * B[k][n] + bias[n] ) over 128-pixel tiles of a crop.
// grid = (tile groups, crops), 288 threads: warps 0-7 = two consumer warpgroups (warpgroup g owns pixels 64 g .. 64 g + 63
// of every tile: wgmma into registers, then the epilogue on its own rows), warp 8 = TMA producer.
// ------------------------------------------------------------------------------------------------------------------
constexpr int GEMM_THREADS = 288;

struct GemmTcArgs {
    CUtensorMap map_hi[2], map_lo[2];   // A sources: box (64 pixels, 2, kc planes, 1 crop)
    int src_planes[2];                  // planes (K / 8) per source
    int src_kc[2];                      // planes per ring chunk (2, 4 or 8) = the box's plane extent
    int n_src;
    int rows_per_tile;                  // 128 / W
    int tiles_per_crop, tiles_per_cta;
    int n_stage;                        // ring depth
    // B: rows [0, gate_rows) are built in the kernel as  gate[b][c] * w3[c][n]  (row = b * midp + c), the rest is copied
    const bf16* b_packed;               // [K8][2*NP][8] packed [hi | lo]; rows below gate_rows are ignored
    int K8;                             // total planes of K
    int N, NP;                          // real / padded (multiple of 16) output channels
    const float* bias;                  // [NP]
    int relu;
    // ChannelGate folded into conv3: the first 4 * midp rows of B come per crop from k_gates_tc (null: no gate)
    const bf16* bfold;                  // [crops][4 * midp / 8][2 * NP][8]
    int midp, HW;
    int slot_bytes;                     // ring slot: hi planes then lo planes (slot_bytes / 2 each)
    // outputs
    bf16* out_hi; bf16* out_lo;         // planes [crops][NP/8][H][W][8] (or pooled [..][H/2][W/2][8]); may be null
    float* out_f32;                     // [crops][HW][N] float32 NHWC copy (may be null)
    int pool;                           // 1: 2x2 average pool in the epilogue (W = tile width)
    int pool2;                          // 1: 2x2 average pool on the SECOND GEMM's output (transition fused behind a block)
    int W;
    // second GEMM on the fresh output tile: out2 = relu(out * B2 + bias2)
    const bf16* b2_packed;              // [NP/8][2*NP2][8] (null: none)
    const float* bias2;
    int N2, NP2;
    bf16* out2_hi; bf16* out2_lo;
    // head fused behind conv5 (one 128-pixel tile per crop): global average pool over the tile, fc (+ folded BatchNorm1d)
    // + ReLU, L2 normalisation, scatter to the caller's row (base_backend.py:197-207, osnet.py:404-421)
    const float* head_w;                // [N][head_feat] (null: no head)
    const float* head_b;                // [head_feat]
    int head_feat;
};
// per-call part of the fused head: the chunk's crop descriptors (out_row) and the caller's feature matrix
struct GemmHeadIO {
    const CropDesc* crops;
    float* out;
    int out_ld;
};

struct GemmSmem {
    size_t b, b2, ring, a2, f, gate, total;
};
inline GemmSmem gemm_smem_layout(int K8, int NP, int NP2, int n_stage, bool tail, bool pool, int slot_bytes, bool pool2 = false) {
    GemmSmem s{};
    size_t o = 0;
    s.b = o; o += (size_t)K8 * 2 * NP * 16;
    s.b2 = o; if (tail) o += (size_t)(NP / 8) * 2 * NP2 * 16;
    o = (o + 127) & ~(size_t)127;
    s.ring = o; o += (size_t)n_stage * slot_bytes;
    s.a2 = o;
    if (tail) {
        size_t a2 = (size_t)2 * (NP / 8) * 128 * 16;
        if (pool2) a2 = a2 > (size_t)128 * (NP2 + 4) * 4 ? a2 : (size_t)128 * (NP2 + 4) * 4;
        o += a2;
    }
    s.f = pool2 ? s.a2 : o;
    if (pool) o += (size_t)128 * (NP + 4) * 4;
    s.gate = o; o += 4 * 32 * 4 + 64;
    s.total = o + 128;
    return s;
}

// Epilogue modes of k_gemm_tc (compile time, with the output widths NP and NP2): bias (+ ReLU) -> planes / float32 NHWC;
// the same with a 2x2 average pool; a second GEMM on the fresh tile (tail) -> planes; the tail with its output pooled
// (a transition fused behind a block); conv5 + the fused head.
enum GemmMode { GM_PLAIN, GM_POOL, GM_TAIL, GM_TAIL_POOL2, GM_HEAD };

// CTAs per SM an instance is compiled for: two (<= 112 registers per thread) where the B operand and a >= 2-deep ring of
// the plan's launches fit half of the SM's shared memory.  One for the combine GEMMs of stages 3 and 4 (B alone is
// 72-128 KB) and for conv5 + head (at 112 registers it spills).  The plan asks the occupancy calculator either way.
template <int NP, int NP2, int MODE>
constexpr int gemm_min_ctas() {
    return NP == 128 || ((MODE == GM_TAIL || MODE == GM_TAIL_POOL2) && NP >= 96) ? 1 : 2;
}

template <int NP, int NP2, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, (gemm_min_ctas<NP, NP2, MODE>()))
    k_gemm_tc(const __grid_constant__ GemmTcArgs a, const int* __restrict__ d_n, int off, int cap, const GemmSmem L, const GemmHeadIO hio) {
    constexpr bool tail = MODE == GM_TAIL || MODE == GM_TAIL_POOL2, pool = MODE == GM_POOL, pool2 = MODE == GM_TAIL_POOL2;
    static_assert(NP % 16 == 0 && NP >= 16 && NP <= 128, "NP: 16 .. 128 output channels");
    static_assert(tail ? (NP2 % 16 == 0 && NP2 >= 16 && NP2 <= 128) : NP2 == 0, "NP2: the tail's output channels");
    constexpr int NACC = (NP2 > NP ? NP2 : NP) / 2;              // accumulator registers per thread (m64nN: N / 2)
    const int n = blockIdx.y;
    if (n >= tc_chunk_count(d_n, off, cap)) return;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_full[4], bar_empty[4], bar_w;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile0 = blockIdx.x * a.tiles_per_cta;
    const int tile1 = min(tile0 + a.tiles_per_cta, a.tiles_per_crop);
    unsigned char* sB = smem + L.b;
    unsigned char* sB2 = smem + L.b2;
    unsigned char* sRing = smem + L.ring;
    unsigned char* sA2 = smem + L.a2;
    float* sF = reinterpret_cast<float*>(smem + L.f);

    if (threadIdx.x == 0) {
        for (int i = 0; i < a.n_stage; ++i) { um::mbar_init(&bar_full[i], 1); um::mbar_init(&bar_empty[i], 2); }
        um::mbar_init(&bar_w, 1);
        um::fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ================= TMA producer =================
        if (lane == 0) {
            {   // packed weights (everything below the gate-folded rows, and the tail's B) by bulk async copies
                const uint32_t first = (uint32_t)((a.bfold ? 4 * a.midp : 0) / 8) * 2u * NP * 16u, total = (uint32_t)a.K8 * 2u * NP * 16u;
                const uint32_t b2 = tail ? (uint32_t)(NP / 8) * 2u * NP2 * 16u : 0u;
                um::mbar_expect_tx(&bar_w, total + b2);
                if (first) um::bulk_g2s(sB, reinterpret_cast<const unsigned char*>(a.bfold) + (size_t)n * first, first, &bar_w);
                if (total > first) um::bulk_g2s(sB + first, reinterpret_cast<const unsigned char*>(a.b_packed) + first, total - first, &bar_w);
                if (b2) um::bulk_g2s(sB2, a.b2_packed, b2, &bar_w);
            }
            uint32_t it = 0;
            for (int tile = tile0; tile < tile1; ++tile) {
                for (int s = 0; s < a.n_src; ++s) {
                    const int kc = a.src_kc[s];
                    for (int p0 = 0; p0 < a.src_planes[s]; p0 += kc, ++it) {
                        const uint32_t slot = it % (uint32_t)a.n_stage, ph = (it / (uint32_t)a.n_stage) & 1u;
                        um::mbar_wait(&bar_empty[slot], ph ^ 1u);
                        unsigned char* dst = sRing + (size_t)slot * a.slot_bytes;
                        um::mbar_expect_tx(&bar_full[slot], (uint32_t)kc * 128u * 16u * 2u);
                        um::tma_load_4d(dst, &a.map_hi[s], 0, tile * 2, p0, n, &bar_full[slot]);
                        um::tma_load_4d(dst + a.slot_bytes / 2, &a.map_lo[s], 0, tile * 2, p0, n, &bar_full[slot]);
                    }
                }
            }
        }
        return;
    }

    // ================= consumer warpgroups =================
    const int et = threadIdx.x;                                 // 0..255
    const int wg = warp >> 2;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // pixel of the tile of accumulator rows h = 0; h = 1 is row + 8
    const int cq = 2 * (lane & 3);                              // first of the two columns of an 8-column group
    const uint32_t lbo_b = 2u * NP * 16u, lo_off = (uint32_t)NP * 16u;   // a K plane of B = NP rows W_hi, then NP rows W_lo
    um::mbar_wait(&bar_w, 0);
    float acc[NACC];
    uint32_t it = 0;
    for (int tile = tile0; tile < tile1; ++tile) {
        uint32_t kplane = 0, first = 1;
        uint32_t held = 0;                                      // slot of the previous chunk, whose MMAs may still run
        // one commit group per k-step (two planes, three MMAs): the next k-step is issued before the previous one has
        // drained, and a ring slot goes back to the producer once the last group that reads it has completed.  Every
        // group accumulates into the same registers in issue order, which wgmma orders by itself; nothing else touches
        // acc until the final wait.  (The MMAs sit unconditionally in the loop body: a conditional wgmma with groups in
        // flight makes ptxas serialise them.)
        for (int s = 0; s < a.n_src; ++s) {
            const int kc = a.src_kc[s];
            for (int p0 = 0; p0 < a.src_planes[s]; p0 += kc, ++it) {
                const uint32_t slot = it % (uint32_t)a.n_stage, ph = (it / (uint32_t)a.n_stage) & 1u;
                um::mbar_wait(&bar_full[slot], ph);
                const uint32_t ah = um::smem_u32(sRing + (size_t)slot * a.slot_bytes) + (uint32_t)wg * 1024u, al = ah + a.slot_bytes / 2;
                for (int ks = 0; ks < kc / 2; ++ks) {
                    const uint32_t bb = um::smem_u32(sB) + (kplane + 2 * ks) * lbo_b;
                    const uint64_t xh = um::make_desc(ah + ks * 2 * 2048u, 2048u, 128), xl = um::make_desc(al + ks * 2 * 2048u, 2048u, 128);
                    um::wg_fence();
                    um::mma<NP, false>(acc, xh, bb, lbo_b, 128, first ? 0u : 1u);      // A_hi W_hi
                    um::mma<NP, false>(acc, xl, bb, lbo_b, 128, 1u);                   // A_lo W_hi
                    um::mma<NP, false>(acc, xh, bb + lo_off, lbo_b, 128, 1u);          // A_hi W_lo
                    first = 0;
                    um::wg_commit();
                    um::wg_wait<1>();                           // the previous k-step's group has completed
                    if (ks == 0 && kplane > 0 && (et & 127) == 0) mbar_arrive(&bar_empty[held]);   // so has the previous chunk
                }
                held = slot;
                kplane += kc;
            }
        }
        um::wg_wait<0>();
        um::wg_fence_acc<NACC>(acc);
        if ((et & 127) == 0) mbar_arrive(&bar_empty[held]);
        if constexpr (MODE == GM_HEAD) {
            // ---- conv5 + head: the tile is the whole 16 x 8 map.  Column sums over the 128 pixels: the two rows of a
            // thread, a butterfly over the 8 row groups of a warp, the 8 warps through shared memory (the ring, once
            // both warpgroups' MMAs have read their last slot; the producer has no further chunk to load) ----
            um::bar_sync(1, 256);
            float* part = reinterpret_cast<float*>(sRing);          // [8][NP]
            float* pooled = part + 8 * NP;                          // [NP]
            float* red = pooled + NP;                               // [8]
            float* feat = red + 8;                                  // [head_feat]
#pragma unroll
            for (int i = 0; i < NP / 8; ++i) {
                const int c = 8 * i + cq;
                const float2 b = *reinterpret_cast<const float2*>(a.bias + c);
                float o0 = fmaxf(acc[4 * i] + b.x, 0.f) + fmaxf(acc[4 * i + 2] + b.x, 0.f);
                float o1 = fmaxf(acc[4 * i + 1] + b.y, 0.f) + fmaxf(acc[4 * i + 3] + b.y, 0.f);
#pragma unroll
                for (int sh = 4; sh < 32; sh <<= 1) {
                    o0 += __shfl_xor_sync(0xffffffffu, o0, sh);
                    o1 += __shfl_xor_sync(0xffffffffu, o1, sh);
                }
                if (lane < 4) *reinterpret_cast<float2*>(part + warp * NP + c) = make_float2(o0, o1);
            }
            um::bar_sync(1, 256);
            for (int c = et; c < NP; c += 256)
                pooled[c] = (((part[c] + part[NP + c]) + (part[2 * NP + c] + part[3 * NP + c])) +
                             ((part[4 * NP + c] + part[5 * NP + c]) + (part[6 * NP + c] + part[7 * NP + c]))) / 128.f;
            um::bar_sync(1, 256);
            const int FEAT = a.head_feat, C = a.N;
            float sq = 0.f;
            for (int f = et; f < FEAT; f += 256) {
                float t[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                int c = 0;
                for (; c + 8 <= C; c += 8) {
#pragma unroll
                    for (int u = 0; u < 8; ++u) t[u] = fmaf(pooled[c + u], a.head_w[(size_t)(c + u) * FEAT + f], t[u]);
                }
                for (; c < C; ++c) t[0] = fmaf(pooled[c], a.head_w[(size_t)c * FEAT + f], t[0]);
                float sv = a.head_b[f] + (((t[0] + t[1]) + (t[2] + t[3])) + ((t[4] + t[5]) + (t[6] + t[7])));
                sv = fmaxf(sv, 0.f);
                feat[f] = sv;
                sq = fmaf(sv, sv, sq);
            }
#pragma unroll
            for (int sh = 16; sh > 0; sh >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, sh);
            if (lane == 0) red[warp] = sq;
            um::bar_sync(1, 256);
            float tot = 0.f;
            for (int w = 0; w < 8; ++w) tot += red[w];
            const float nrm = sqrtf(tot);
            float* dst = hio.out + (size_t)hio.crops[off + n].out_row * hio.out_ld;
            for (int f = et; f < FEAT; f += 256) dst[f] = feat[f] / nrm;
            um::bar_sync(1, 256);                                  // part / pooled are rewritten by the next tile
        } else {
            // ---- epilogue: bias (+ ReLU) on the thread's two rows x (2 columns per 8-column group) ----
#pragma unroll
            for (int i = 0; i < NP / 8; ++i) {
                const int c = 8 * i + cq;
                const float2 b = *reinterpret_cast<const float2*>(a.bias + c);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = row + 8 * h, px = tile * 128 + m;
                    float o0 = acc[4 * i + 2 * h] + b.x, o1 = acc[4 * i + 2 * h + 1] + b.y;
                    if (a.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                    if (a.out_f32) {
                        float* dst = a.out_f32 + ((size_t)n * a.HW + px) * a.N + c;
                        if (c + 1 < a.N) *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
                        else if (c < a.N) dst[0] = o0;
                    }
                    if constexpr (pool) {
                        *reinterpret_cast<float2*>(sF + (size_t)m * (NP + 4) + c) = make_float2(o0, o1);
                    } else if (a.out_hi || tail) {
                        uint32_t hv, lv;
                        um::split2(o0, o1, hv, lv);
                        if (a.out_hi) {
                            const size_t e = (((size_t)n * (NP / 8) + i) * a.HW + px) * 4 + (lane & 3);
                            reinterpret_cast<uint32_t*>(a.out_hi)[e] = hv;
                            reinterpret_cast<uint32_t*>(a.out_lo)[e] = lv;
                        }
                        if constexpr (tail) {
                            *reinterpret_cast<uint32_t*>(sA2 + ((size_t)i * 128 + m) * 16 + (lane & 3) * 4) = hv;
                            *reinterpret_cast<uint32_t*>(sA2 + ((size_t)(NP / 8 + i) * 128 + m) * 16 + (lane & 3) * 4) = lv;
                        }
                    }
                }
            }
            // 2x2 average pool of the tile in sF (rows_per_tile x W, row stride NPx + 4) -> (rows/2 x W/2) planes;
            // (a + b + c + d) * 0.25, a=(y,x) b=(y,x+1) c=(y+1,x) d=(y+1,x+1)
            auto pool_store = [&](const int NPx, bf16* o_hi, bf16* o_lo) {
                um::bar_sync(1, 256);
                const int Wt = a.W, OW = Wt / 2, OHt = a.rows_per_tile / 2;
                const int items = OHt * OW * (NPx / 8);
                const int OHW = a.HW / 4;
                for (int e = et; e < items; e += 256) {
                    const int pp = e % (OHt * OW), c8 = e / (OHt * OW);
                    const int oy = pp / OW, ox = pp - oy * OW;
                    const float* f0 = sF + (size_t)((2 * oy) * Wt + 2 * ox) * (NPx + 4) + c8 * 8;
                    const float* f1 = f0 + (NPx + 4);
                    const float* f2 = f0 + (size_t)Wt * (NPx + 4);
                    const float* f3 = f2 + (NPx + 4);
                    uint32_t h[4], l[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float x0 = (f0[2 * j] + f1[2 * j] + f2[2 * j] + f3[2 * j]) * 0.25f;
                        const float x1 = (f0[2 * j + 1] + f1[2 * j + 1] + f2[2 * j + 1] + f3[2 * j + 1]) * 0.25f;
                        um::split2(x0, x1, h[j], l[j]);
                    }
                    const int opx = (tile * OHt + oy) * OW + ox;
                    const size_t o = ((size_t)n * (NPx / 8) + c8) * OHW + opx;
                    reinterpret_cast<uint4*>(o_hi)[o] = make_uint4(h[0], h[1], h[2], h[3]);
                    reinterpret_cast<uint4*>(o_lo)[o] = make_uint4(l[0], l[1], l[2], l[3]);
                }
                um::bar_sync(1, 256);   // sF is rewritten by the next tile
            };
            if constexpr (pool) pool_store(NP, a.out_hi, a.out_lo);
            if constexpr (tail) {
                // the fresh tile (hi | lo planes in sA2) is the A operand of the second GEMM: a warpgroup's MMAs read only the
                // 64 rows it wrote itself
                um::fence_async_smem();
                um::bar_sync(2 + wg, 128);
                const uint32_t lbo_b2 = 2u * NP2 * 16u, lo2 = (uint32_t)NP2 * 16u;
                const uint32_t ah = um::smem_u32(sA2) + (uint32_t)wg * 1024u, al = ah + (uint32_t)(NP / 8) * 2048u;
                um::wg_fence();
                for (int ks = 0; ks < NP / 16; ++ks) {
                    const uint32_t bb = um::smem_u32(sB2) + ks * 2 * lbo_b2;
                    const uint64_t xh = um::make_desc(ah + ks * 2 * 2048u, 2048u, 128), xl = um::make_desc(al + ks * 2 * 2048u, 2048u, 128);
                    um::mma<NP2, false>(acc, xh, bb, lbo_b2, 128, ks > 0);
                    um::mma<NP2, false>(acc, xl, bb, lbo_b2, 128, 1u);
                    um::mma<NP2, false>(acc, xh, bb + lo2, lbo_b2, 128, 1u);
                }
                um::wg_commit();
                um::wg_wait<0>();
                um::wg_fence_acc<NACC>(acc);
                if constexpr (pool2) um::bar_sync(1, 256);             // sF aliases sA2: both warpgroups' MMAs have read it
#pragma unroll
                for (int i = 0; i < NP2 / 8; ++i) {
                    const int c = 8 * i + cq;
                    const float2 b = *reinterpret_cast<const float2*>(a.bias2 + c);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int m = row + 8 * h, px = tile * 128 + m;
                        const float o0 = fmaxf(acc[4 * i + 2 * h] + b.x, 0.f), o1 = fmaxf(acc[4 * i + 2 * h + 1] + b.y, 0.f);
                        if constexpr (pool2) {
                            *reinterpret_cast<float2*>(sF + (size_t)m * (NP2 + 4) + c) = make_float2(o0, o1);
                        } else {
                            uint32_t hv, lv;
                            um::split2(o0, o1, hv, lv);
                            const size_t e = (((size_t)n * (NP2 / 8) + i) * a.HW + px) * 4 + (lane & 3);
                            reinterpret_cast<uint32_t*>(a.out2_hi)[e] = hv;
                            reinterpret_cast<uint32_t*>(a.out2_lo)[e] = lv;
                        }
                    }
                }
                if constexpr (pool2) pool_store(NP2, a.out2_hi, a.out2_lo);
            }
        }
    }
}

// the instances the plan of OSNet_x0_25 launches (both launch lists); a layout without one is refused at plan build
typedef void (*GemmKernel)(GemmTcArgs, const int*, int, int, GemmSmem, GemmHeadIO);
struct GemmInstance { int NP, NP2, mode; GemmKernel fn; };
#define BMB_GEMM(np, np2, mode) {np, np2, mode, k_gemm_tc<np, np2, mode>}
static const GemmInstance kGemmInstances[] = {
    BMB_GEMM(16, 0, GM_PLAIN), BMB_GEMM(32, 0, GM_PLAIN),     // conv1 of every block
    BMB_GEMM(64, 0, GM_PLAIN), BMB_GEMM(96, 0, GM_PLAIN),     // combine without a tail (diagnostic list)
    BMB_GEMM(128, 0, GM_PLAIN),                               // combine of the last block; conv5 (diagnostic list)
    BMB_GEMM(64, 0, GM_POOL), BMB_GEMM(96, 0, GM_POOL),       // unfused transitions (diagnostic list)
    BMB_GEMM(64, 16, GM_TAIL), BMB_GEMM(96, 32, GM_TAIL), BMB_GEMM(128, 32, GM_TAIL),   // combine + next conv1
    BMB_GEMM(64, 64, GM_TAIL_POOL2), BMB_GEMM(96, 96, GM_TAIL_POOL2),                   // combine + transition
    BMB_GEMM(128, 0, GM_HEAD),                                // conv5 + head
};
#undef BMB_GEMM
inline GemmKernel gemm_instance(int NP, int NP2, int mode) {
    for (const GemmInstance& g : kGemmInstances)
        if (g.NP == NP && g.NP2 == NP2 && g.mode == mode) return g.fn;
    return nullptr;
}


// ------------------------------------------------------------------------------------------------------------------
// k_front_tc: detection crop -> OpenCV-exact bilinear resize (uint8) -> 7x7 stride-2 stem (+BN, ReLU) on the tensor
// cores -> 3x3 stride-2 max pool -> split planes P [crops][2][64][32][8].  Replaces get_crops + ConvLayer + maxpool
// (reid/backends/base_backend.py:148-195, reid/backbones/osnet.py:27-60,380-384) and the float32 blob / stem tensors
// of round 1 (82 MB + 109 MB per frame written and re-read).
//
// * The resized crop is integer valued (cv2.resize on uint8): it is EXACT in BF16, so the A operand has no low part.
//   The input normalisation is folded into the weights, W' = w / (255 std), and into a bias table,
//   b' = b - sum_{taps inside the image} w mean / std, one entry per (row class, column class) of the output pixel
//   (zero padding applies to the NORMALISED input: at the border some taps do not contribute their mean term).
// * A CTA = (crop, strip of 8 pooled columns): the 39 input columns it needs are staged column-major with 4 channels
//   per pixel, [col][padded row][R G B 0] BF16 (8 B per pixel, 2112 B per column).  The 7 vertical taps x 4 channels of
//   output row oy of one input column are then the 64 contiguous bytes at 16 * oy: a "Toeplitz" A operand with
//   LBO = 16 B, SBO = 128 B (overlapping rows; the stem parity tests of tests/test_gpu_reid.py pin it).  One M tile = the
//   128 output rows of one stem column; K = 7 kx x (8 taps x 4 channels) = 14 K steps of 16; B = [W'_hi | W'_lo].
// * Warpgroup g owns output rows 64 g .. 64 g + 63 of every stem column (one m64n32 accumulator): the pool's horizontal
//   maximum runs over consecutive stem columns in the same thread's registers, the vertical one over rows staged in
//   shared memory (up to 4 pooled columns x 128 rows x 16 channels per batch of 8 stem columns).
// grid = (4 strips, crops), 256 threads (two warpgroups), 130 KB shared memory.
// ------------------------------------------------------------------------------------------------------------------
struct FrontTcArgs {
    const uint8_t* images;
    size_t image_stride;
    int rows, cols;
    const void* crops;                  // CropDesc[] (engine.h): x1, y1, x2, y2, image, out_row
    const bf16* w;                      // [7 kx][4 k8][32 n'][8]: n' < 16 hi, n' >= 16 lo
    const float* bias_tab;              // [4 row classes][4 column classes][16]
    bf16* p_hi;
    bf16* p_lo;
    float* dbg_crop;                    // diagnostics: resized crop [crops][256][128][3] (RGB) as float, or null
    int pad_mode;                       // 0 resize, 1 resize_pad (aspect-preserving resize, ImageNet-mean border)
};
struct FrontCrop { float x1, y1, x2, y2; int image, out_row; };

constexpr int FR_COLS = 39, FR_ROWS = 264, FR_CS = FR_ROWS * 8 + 16;     // staged columns, padded rows, bytes per column (+16: bank spread)
constexpr int FR_A_BYTES = FR_COLS * FR_CS;
constexpr int FR_W_BYTES = 7 * 4 * 32 * 16;
constexpr int FR_H_BYTES = 4 * 128 * 16 * 4;                                // horizontally pooled rows of one batch
constexpr size_t FR_SMEM = FR_A_BYTES + FR_W_BYTES + FR_H_BYTES + 128;

__device__ __forceinline__ void fr_coeff(int d, int src_n, double scale, bool clamp, int& idx, int& a0, int& a1) {
    float f = (float)(((double)d + 0.5) * scale - 0.5);
    int s = (int)floorf(f);
    f = f - (float)s;
    if (clamp) {
        if (s < 0) { s = 0; f = 0.f; }
        if (s >= src_n - 1) { s = src_n - 1; f = 0.f; }
    }
    idx = s;
    a0 = (int)rintf((1.0f - f) * 2048.0f);
    a1 = (int)rintf(f * 2048.0f);
}

__global__ void __launch_bounds__(256, 1) k_front_tc(const FrontTcArgs a, const int* __restrict__ d_n, int off, int cap) {
    const int n = blockIdx.y;
    if (n >= tc_chunk_count(d_n, off, cap)) return;
    const int strip = blockIdx.x;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ int xi[128], xa0[128], xa1[128], yi[256], ya0[256], ya1[256];
    __shared__ __align__(16) float sBias[4 * 4 * 16];
    unsigned char* sA = smem;
    unsigned char* sW = smem + FR_A_BYTES;
    float* sH = reinterpret_cast<float*>(smem + FR_A_BYTES + FR_W_BYTES);   // [4 pooled columns][128 rows][16 channels]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const FrontCrop cd = reinterpret_cast<const FrontCrop*>(a.crops)[off + n];
#ifdef BMB_TC_CLOCKS
    long long fk[16];
    int nfk = 0;
#define FCK() do { if (threadIdx.x == 0 && nfk < 16) fk[nfk++] = clock64(); } while (0)
#else
#define FCK() do { } while (0)
#endif
    FCK();

    // box.round().astype(int): round half to even; clip to the frame (base_backend.py:160-175)
    const int x1 = (int)rintf(cd.x1), y1 = (int)rintf(cd.y1), x2 = (int)rintf(cd.x2), y2 = (int)rintf(cd.y2);
    const int cx1 = max(0, x1), cy1 = max(0, y1), cx2 = min(a.cols, x2), cy2 = min(a.rows, y2);
    const bool valid = cx2 > cx1 && cy2 > cy1;
    const int sw = cx2 - cx1, sh = cy2 - cy1;
    // resize_pad (preprocessing.py:21-45): scale = min(W / w, H / h); new = int(size * scale); centred, ImageNet-mean border
    int nw = 128, nh = 256, pl = 0, pt = 0;
    if (valid && a.pad_mode) {
        const double sc = fmin(128.0 / (double)sw, 256.0 / (double)sh);
        nw = max(1, (int)((double)sw * sc));
        nh = max(1, (int)((double)sh * sc));
        pl = (128 - nw) / 2;
        pt = (256 - nh) / 2;
    }
    if (valid) {
        const double sx = 1.0 / ((double)nw / (double)sw), sy = 1.0 / ((double)nh / (double)sh);
        for (int d = threadIdx.x; d < nw; d += 256) fr_coeff(d, sw, sx, true, xi[d], xa0[d], xa1[d]);
        for (int d = threadIdx.x; d < nh; d += 256) fr_coeff(d, sh, sy, false, yi[d], ya0[d], ya1[d]);
    }
    for (int e = threadIdx.x; e < FR_A_BYTES / 16; e += 256) reinterpret_cast<uint4*>(sA)[e] = make_uint4(0u, 0u, 0u, 0u);
    for (int e = threadIdx.x; e < FR_W_BYTES / 16; e += 256) reinterpret_cast<uint4*>(sW)[e] = reinterpret_cast<const uint4*>(a.w)[e];
    for (int e = threadIdx.x; e < 256; e += 256) sBias[e] = a.bias_tab[e];
    __syncthreads();
    FCK();
    const int xin0 = 32 * strip - 5;                               // input column of staged column 0
    if (valid) {
        // cv2.resize(INTER_LINEAR) on uint8: 11-bit coefficients, horizontal pass in int32, vertical
        // (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2  (bit-exact; tests pin it against OpenCV)
        const uint8_t* img = a.images + (size_t)cd.image * a.image_stride;
        // lanes run along the staged columns of one output row: neighbouring lanes read neighbouring source pixels of the
        // same two source rows (coalesced); four pixels per thread are in flight at once (the loop is latency-bound:
        // table lookups -> 12 byte loads -> integer arithmetic -> one 8-byte shared store)
        for (int base = threadIdx.x; base < 40 * 256; base += 4 * 256) {
            int h0[4][3], h1[4][3], bb0[4], bb1[4], so[4];
            bool ok[4], border[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int p = base + u * 256;
                const int dy = p / 40, lc = p - dy * 40;
                const int dx = xin0 + lc;
                ok[u] = p < 40 * 256 && lc < FR_COLS && dx >= 0 && dx < 128;
                const int ry = dy - pt, rx = dx - pl;             // position in the resized patch (resize: the crop itself)
                border[u] = rx < 0 || rx >= nw || ry < 0 || ry >= nh;
                const int dxc = min(max(rx, 0), nw - 1), dyc = min(max(ry, 0), nh - 1);
                const int sx0 = xi[dxc], sx1 = min(sx0 + 1, sw - 1);
                const int r0 = min(max(yi[dyc], 0), sh - 1), r1 = min(max(yi[dyc] + 1, 0), sh - 1);
                const uint8_t* p0 = img + ((size_t)(cy1 + r0) * a.cols + cx1) * 3;
                const uint8_t* p1 = img + ((size_t)(cy1 + r1) * a.cols + cx1) * 3;
                const int a0 = xa0[dxc], a1 = xa1[dxc];
                bb0[u] = ya0[dyc]; bb1[u] = ya1[dyc];
                so[u] = lc * FR_CS + (min(dy, 255) + 3) * 8;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    h0[u][c] = (int)__ldg(p0 + sx0 * 3 + c) * a0 + (int)__ldg(p0 + sx1 * 3 + c) * a1;
                    h1[u][c] = (int)__ldg(p1 + sx0 * 3 + c) * a0 + (int)__ldg(p1 + sx1 * 3 + c) * a1;
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (!ok[u]) continue;
                int v[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const int r = (((bb0[u] * (h0[u][c] >> 4)) >> 16) + ((bb1[u] * (h1[u][c] >> 4)) >> 16) + 2) >> 2;
                    v[c] = min(max(r, 0), 255);
                }
                if (border[u]) { v[0] = 104; v[1] = 116; v[2] = 124; }      // IMAGENET_MEAN_BGR
                // BGR source -> RGB network order; integers 0..255 are exact in BF16
                const __nv_bfloat162 rg = __floats2bfloat162_rn((float)v[2], (float)v[1]);
                const __nv_bfloat162 b_ = __floats2bfloat162_rn((float)v[0], 0.f);
                *reinterpret_cast<uint2*>(sA + so[u]) = make_uint2(*reinterpret_cast<const uint32_t*>(&rg), *reinterpret_cast<const uint32_t*>(&b_));
                if (a.dbg_crop) {
                    const int p = base + u * 256;
                    const int dy = p / 40, dx = xin0 + (p - dy * 40);
                    float* o = a.dbg_crop + (((size_t)n * 256 + dy) * 128 + dx) * 3;
                    o[0] = (float)v[2]; o[1] = (float)v[1]; o[2] = (float)v[0];
                }
            }
        }
    } else if (a.dbg_crop) {
        for (int p = threadIdx.x; p < 40 * 256; p += 256) {
            const int dy = p / 40, lc = p - dy * 40;
            const int dx = xin0 + lc;
            if (lc < FR_COLS && dx >= 0 && dx < 128) {
                float* o = a.dbg_crop + (((size_t)n * 256 + dy) * 128 + dx) * 3;
                o[0] = 0.f; o[1] = 0.f; o[2] = 0.f;
            }
        }
    }
    um::fence_async_smem();
    __syncthreads();
    FCK();

    // stem columns of this strip: j = 0..16  <->  ox = 16 * strip - 1 + j  (ox = -1 does not exist: zero)
    const int wg = warp >> 2;
    const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // output rows oy = row (h = 0) and row + 8 (h = 1)
    const int cq = 2 * (lane & 3);                                 // channels 8 i + cq + e, i, e in {0, 1}
    int rcl[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int oy = row + 8 * h;
        rcl[h] = oy == 0 ? 0 : (oy == 1 ? 1 : (oy == 127 ? 3 : 2));
    }
    float prev1[2][4], prev2[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < 4; ++c) { prev1[h][c] = 0.f; prev2[h][c] = 0.f; }
    const uint32_t sa = um::smem_u32(sA) + (uint32_t)wg * 1024u, sw_ = um::smem_u32(sW);
    for (int j0 = 0; j0 < 17; j0 += 8) {
        const int j1 = min(j0 + 8, 17);
        // ---- per stem column: MMAs, bias + ReLU, horizontal 3-max over consecutive stem columns (registers) ----
        for (int j = j0; j < j1; ++j) {
            const int ox = 16 * strip - 1 + j;
            float v[2][4];
            if (ox >= 0) {
                float acc[16];
                um::wg_fence();
#pragma unroll
                for (int kx = 0; kx < 7; ++kx)
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks)
                        um::mma<32, false>(acc, um::make_desc(sa + (uint32_t)(2 * j + kx) * FR_CS + ks * 32, 16, 128),
                                           sw_ + (uint32_t)(kx * 4 + 2 * ks) * 512u, 512u, 128, (kx | ks) != 0);
                um::wg_commit();
                um::wg_wait_all();
                um::wg_fence_acc<16>(acc);
                const int cc = ox == 0 ? 0 : (ox == 1 ? 1 : (ox == 63 ? 3 : 2));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float* bb = sBias + (rcl[h] * 4 + cc) * 16;
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e)   // [W_hi | W_lo]: channel c is column c plus column c + 16
                            v[h][2 * i + e] = fmaxf(acc[4 * i + 2 * h + e] + acc[4 * (i + 2) + 2 * h + e] + bb[8 * i + cq + e], 0.f);
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c = 0; c < 4; ++c) v[h][c] = 0.f;
            }
            if ((j & 1) == 0 && j >= 2) {                          // ox = 2 px + 1: third column of pooled px = 8 strip + j / 2 - 1
                float* hs = sH + (size_t)(((j - j0) >> 1) & 3) * 128 * 16;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        *reinterpret_cast<float2*>(hs + (row + 8 * h) * 16 + 8 * i + cq) =
                            make_float2(fmaxf(fmaxf(prev2[h][2 * i], prev1[h][2 * i]), v[h][2 * i]),
                                        fmaxf(fmaxf(prev2[h][2 * i + 1], prev1[h][2 * i + 1]), v[h][2 * i + 1]));
            }
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int c = 0; c < 4; ++c) { prev2[h][c] = prev1[h][c]; prev1[h][c] = v[h][c]; }
        }
        __syncthreads();
        // pooled columns finished in this batch: j = 2, 4, 6 (batch 0) -> slots 1, 2, 3;  batch 1 (j0 = 8): j = 8, 10, 12,
        // 14 -> slots 0..3;  batch 2: j = 16 -> slot 0
        const int s_first = j0 == 0 ? 1 : 0, s_last = j0 == 0 ? 3 : (j0 == 8 ? 3 : 0);
        // ---- vertical 3-max over rows (oy - 1, oy, oy + 1), oy = 2 py; one item = (slot, py, 8 channels) ----
        const int items = (s_last - s_first + 1) * 64 * 2;
        for (int e = threadIdx.x; e < items; e += 256) {
            const int s = s_first + (e >> 7), py = (e >> 1) & 63, half = e & 1;
            const float* hs = sH + (size_t)s * 128 * 16 + half * 8;
            const int oy = 2 * py;
            float m[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const float up = oy > 0 ? hs[(oy - 1) * 16 + c] : 0.f;
                m[c] = fmaxf(fmaxf(up, hs[oy * 16 + c]), hs[(oy + 1) * 16 + c]);
            }
            const int px = 8 * strip + (j0 + 2 * s) / 2 - 1;
            uint32_t h4[4], l4[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) um::split2(m[2 * c], m[2 * c + 1], h4[c], l4[c]);
            const size_t o = (((size_t)n * 2 + half) * 64 + py) * 32 + px;
            reinterpret_cast<uint4*>(a.p_hi)[o] = make_uint4(h4[0], h4[1], h4[2], h4[3]);
            reinterpret_cast<uint4*>(a.p_lo)[o] = make_uint4(l4[0], l4[1], l4[2], l4[3]);
        }
        __syncthreads();                                            // sH is reused by the next batch
        FCK();
    }
#ifdef BMB_TC_CLOCKS
    if (threadIdx.x == 0 && n == 5) {
        printf("front strip %d: setup %lld resize %lld |", strip, fk[1] - fk[0], fk[2] - fk[1]);
        for (int i = 3; i < nfk; ++i) printf(" batch %lld |", fk[i] - fk[i - 1]);
        printf(" total %lld\n", fk[nfk - 1] - fk[0]);
    }
#endif
}

}  // namespace tcx
}  // namespace bmb
