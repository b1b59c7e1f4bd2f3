// tracker_engine.cu -- host side of the device-resident tracker: memory, launches, and the kernels that wrap
// tracker_core.cuh.  One Engine owns `n_streams` independent trackers resident on one GPU; a frame for all
// of them is: H2D (dets [+ embs | frames]) -> [crop list -> ReID] -> appearance prep -> cosine cost (wide
// grid) -> one CTA per stream running the whole association / Kalman / lifecycle -> D2H rows.
//
// Replaces the host loops of BaseTracker.update()/_update_impl (trackers/basetracker.py:120-147,
// bytetrack.py:259-403, botsort.py:177-249) and the native Update() (native/cpp/trackers/botsort/src/
// tracker.cpp:329-498) behind the same C ABI.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "engine.h"
#include "host_stage.h"
#include "tracker_core.cuh"
#include "tracker_layout.h"

namespace bmb {

#define CUDA_OK(expr)                                                                                   \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess)                                                                          \
            throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e));              \
    } while (0)

// ---------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------
// Shared-memory residency for the assignment's dual prices / frontier arrays (they are touched on every step of
// the augmenting-path search); falls back to the HBM scratch of the slab when the capacities are too large.
__host__ __device__ inline size_t lap_smem_bytes(int CT, int CD) {
    return sizeof(double) * ((size_t)CT + 2 * (size_t)CD) + sizeof(int) * (2 * (size_t)CT + 1 + 5 * (size_t)CD) + 16;
}

#ifndef BMB_FRAME_THREADS
#define BMB_FRAME_THREADS 256
#endif
__global__ void __launch_bounds__(BMB_FRAME_THREADS) k_tracker_frame(const TrkCfg cfg, TrkStream* streams, int lap_in_smem) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    TrkStream s = streams[blockIdx.x];
    if (lap_in_smem) {
        const int CT = cfg.cap_tracks, CD = cfg.cap_dets;
        double* pd = reinterpret_cast<double*>(dyn_smem);
        s.lap_u = pd; pd += CT;
        s.lap_v = pd; pd += CD;
        s.lap_spc = pd; pd += CD;
        int* pi = reinterpret_cast<int*>(pd);
        s.lap_x = pi; pi += CT;
        s.csr_ptr = pi; pi += CT + 1;
        s.lap_y = pi; pi += CD;
        s.lap_path = pi; pi += CD;
        s.lap_insc = pi; pi += CD;
        s.lap_tl = pi; pi += CD;
        s.lap_sc = pi;
    }
    tracker_frame(cfg, s);
}

// the appearance EMA of this frame's matched (track, detection) pairs, one warp per pair
__global__ void __launch_bounds__(256) k_feat_ema(const TrkCfg cfg, TrkStream* streams) {
    TrkStream s = streams[blockIdx.y];
    const int pair = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pair >= s.scalars[SC_N_EMA]) return;
    apply_feature_ema(cfg, s, pair);
}

// detection appearance: the reference normalises each high-confidence row twice in place
// (botsort_track.py:58-67 on a fresh STrack); one warp per detection row.
__global__ void __launch_bounds__(256) k_feat_prepare(const TrkCfg cfg, TrkStream* streams, const float* embs) {
    const TrkStream& s = streams[blockIdx.y];
    const int D = min(*s.n_dets, cfg.cap_dets);
    const int F = cfg.feat_dim;
    const int warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (warp >= D) return;
    const float cf = s.dets[warp * 6 + 4];
    if (!((double)cf > cfg.high_thresh)) return;  // only first-round detections carry appearance
    const float* src = embs + ((size_t)blockIdx.y * cfg.cap_dets + warp) * F;
    feat_prepare(src, s.dfeat + (size_t)warp * F, F);
}

// max(0, cosine distance) between every live track's smoothed appearance and every first-round detection,
// float64 accumulate over float32 inputs (scipy cdist semantics, matching.py:85-107).  Tile = 8 track rows x
// 32 detections per CTA, K staged through shared memory in chunks of 64.
constexpr int EMB_TR = 8, EMB_TD = 32, EMB_TK = 64;
__global__ void __launch_bounds__(256) k_embedding_cost(const TrkCfg cfg, TrkStream* streams) {
    const TrkStream& s = streams[blockIdx.z];
    const int D = min(*s.n_dets, cfg.cap_dets);
    const int na = s.scalars[SC_N_ACTIVE], nl = s.scalars[SC_N_LOST];
    const int T = na + nl;
    const int r0 = blockIdx.y * EMB_TR, d0 = blockIdx.x * EMB_TD;
    if (r0 >= T || d0 >= D) return;
    __shared__ float sa[EMB_TR][EMB_TK + 1];
    __shared__ float sb[EMB_TD][EMB_TK + 1];
    __shared__ int slot_of[EMB_TR];
    const int F = cfg.feat_dim;
    const int tr = threadIdx.x / EMB_TD, td = threadIdx.x % EMB_TD;
    if (threadIdx.x < EMB_TR) {
        int r = r0 + threadIdx.x;
        slot_of[threadIdx.x] = r < T ? (r < na ? s.active[r] : s.lost[r - na]) : -1;
    }
    __syncthreads();
    double dot = 0.0, na2 = 0.0, nb2 = 0.0;
    for (int k0 = 0; k0 < F; k0 += EMB_TK) {
        for (int e = threadIdx.x; e < EMB_TR * EMB_TK; e += blockDim.x) {
            int r = e / EMB_TK, k = e % EMB_TK;
            int slot = slot_of[r];
            sa[r][k] = (slot >= 0 && k0 + k < F) ? s.smooth[(size_t)slot * F + k0 + k] : 0.f;
        }
        for (int e = threadIdx.x; e < EMB_TD * EMB_TK; e += blockDim.x) {
            int d = e / EMB_TK, k = e % EMB_TK;
            sb[d][k] = (d0 + d < D && k0 + k < F) ? s.dfeat[(size_t)(d0 + d) * F + k0 + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < EMB_TK; ++k) {
            double x = (double)sa[tr][k], y = (double)sb[td][k];
            dot += x * y; na2 += x * x; nb2 += y * y;
        }
        __syncthreads();
    }
    const int slot = slot_of[tr];
    if (slot >= 0 && d0 + td < D) {
        double cs = dot / (sqrt(na2) * sqrt(nb2));
        if (fabs(cs) > 1.0) cs = cs > 0 ? 1.0 : -1.0;
        double dist = 1.0 - cs;
        dist = dist > 0.0 ? dist : (dist != dist ? dist : 0.0);
        s.embd[(size_t)slot * cfg.cap_dets + d0 + td] = dist;
    }
}

// DeepOCSORT appearance similarity dets_embs @ trk_embs.T (deepocsort.py:391) for every (detection, live slot):
// float32 detection rows x float64 track EMAs, float64 accumulate.  Inside the one-CTA frame kernel this product was
// 7 of the 8 ms of a 256-detection frame; on a wide grid it is microseconds.  Tile = 8 tracks x 32 detections.
__global__ void __launch_bounds__(256) k_docs_embcost(const DocsCfg cfg, DocsStream* streams) {
    const DocsStream& s = streams[blockIdx.z];
    const int D = min(*s.n_dets, cfg.cap_dets);
    const int T = s.scalars[SC_N_ACTIVE];
    const int r0 = blockIdx.y * EMB_TR, d0 = blockIdx.x * EMB_TD;
    if (r0 >= T || d0 >= D) return;
    __shared__ double sa[EMB_TR][EMB_TK + 1];
    __shared__ float sb[EMB_TD][EMB_TK + 1];
    __shared__ int slot_of[EMB_TR];
    const int F = cfg.feat_dim;
    const int tr = threadIdx.x / EMB_TD, td = threadIdx.x % EMB_TD;
    if (threadIdx.x < EMB_TR) slot_of[threadIdx.x] = r0 + threadIdx.x < T ? s.tracks[r0 + threadIdx.x] : -1;
    __syncthreads();
    double dot = 0.0;
    for (int k0 = 0; k0 < F; k0 += EMB_TK) {
        for (int e = threadIdx.x; e < EMB_TR * EMB_TK; e += blockDim.x) {
            const int r = e / EMB_TK, k = e % EMB_TK;
            const int slot = slot_of[r];
            sa[r][k] = (slot >= 0 && k0 + k < F) ? s.emb[(size_t)slot * F + k0 + k] : 0.0;
        }
        for (int e = threadIdx.x; e < EMB_TD * EMB_TK; e += blockDim.x) {
            const int d = e / EMB_TK, k = e % EMB_TK;
            sb[d][k] = (d0 + d < D && k0 + k < F) ? s.embs[(size_t)(d0 + d) * F + k0 + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < EMB_TK; ++k) dot += (double)sb[td][k] * sa[tr][k];
        __syncthreads();
    }
    const int slot = slot_of[tr];
    if (slot >= 0 && d0 + td < D) s.embq[(size_t)(d0 + td) * cfg.cap_tracks + slot] = dot;
}

// CTA-wide augmentation of the dense JV solver (jv_dense.cuh::jv_augment_wide) replaces the one-warp walk on the
// BASELINE config-3 shape (512 detections, 1 500 live tracks) with identical results; the column-owned variant
// (jv_augment_owned, mode 2) goes further.  Mode 3 (the default) is mode 2 plus the two exact shortcuts described at jv_augment_owned
// (no-op band columns walked over, parallel tail of _find_dense).  BOXMOT_B200_JV_WIDE=0/1/2/3 sets the initial
// value, boxmot_b200_jv_dense_mode() changes it (parity tests run every variant).
// 0..2: the older variants; 3: mode 3 with every shortcut; >= 4: raw `mode | feature bits << 2` (bisecting on hardware)
static int jv_mode_value(int m) { return m < 0 ? 0 : (m == 3 ? (3 | (0xF << 2)) : (m > 63 ? 63 : m)); }
static int& jv_wide_flag() {
    static int v = [] {
        const char* e = getenv("BOXMOT_B200_JV_WIDE");
        return jv_mode_value(e ? atoi(e) : 3);
    }();
    return v;
}
static int jv_wide_default() { return jv_wide_flag(); }

// shared-memory residency of the dense JV solver's per-column / per-row state (prices, distances, column list, ...)
__host__ __device__ inline size_t jv_smem_bytes(int MX) {
    return (size_t)MX * (2 * sizeof(double) + 6 * sizeof(int)) + 16;
}

// lapjv's scratch of a stream copy re-pointed into the frame kernel's dynamic shared memory (jv_smem_bytes(MX) bytes)
template <typename St>
__device__ __forceinline__ void jv_scratch_to_smem(St& s, unsigned char* smem, int MX) {
    double* pd = reinterpret_cast<double*>(smem);
    s.lap_v = pd; pd += MX;
    s.lap_spc = pd; pd += MX;
    int* pi = reinterpret_cast<int*>(pd);
    s.lap_x = pi; pi += MX;
    s.lap_y = pi; pi += MX;
    s.lap_path = pi; pi += MX;
    s.lap_tl = pi; pi += MX;
    s.lap_sc = pi; pi += MX;
    s.lap_insc = pi;
}

// Dynamic shared memory for a launch of `frame_kernel` (lapjv's scratch, when it fits) and the kernel's jv_in_smem
// argument: bit 0 = the scratch lives there, the bits above = the dense-JV augmentation mode
template <typename Kernel>
static int jv_launch_setup(Kernel frame_kernel, int cap_tracks, int cap_dets, size_t* smem_bytes) {
    const size_t jb = jv_smem_bytes(cap_tracks > cap_dets ? cap_tracks : cap_dets);
    const bool in_smem = jb <= 200 * 1024;
    if (in_smem && jb > 48 * 1024)
        CUDA_OK(cudaFuncSetAttribute(frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)jb));
    *smem_bytes = in_smem ? jb : 0;
    return (in_smem ? 1 : 0) | (jv_wide_default() << 1);
}

__global__ void __launch_bounds__(256) k_docs_frame(const DocsCfg cfg, DocsStream* streams, int jv_in_smem) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    DocsStream s = streams[blockIdx.x];
    s.jv_wide = jv_in_smem >> 1;
    if (jv_in_smem & 1) {   // jv_scratch_to_smem, written out: at 255 registers with spills, this kernel's allocation moves with the helper
        const int MX = cfg.cap_tracks > cfg.cap_dets ? cfg.cap_tracks : cfg.cap_dets;
        double* pd = reinterpret_cast<double*>(dyn_smem);
        s.lap_v = pd; pd += MX;
        s.lap_spc = pd; pd += MX;
        int* pi = reinterpret_cast<int*>(pd);
        s.lap_x = pi; pi += MX;
        s.lap_y = pi; pi += MX;
        s.lap_path = pi; pi += MX;
        s.lap_tl = pi; pi += MX;
        s.lap_sc = pi; pi += MX;
        s.lap_insc = pi;
    }
    docs_frame(cfg, s);
}

// BoostTrack appearance similarity dets_embs @ trk_embs.T (boosttrack.py:353-358) for every (detection row, live slot):
// float32 rows x float64 track embeddings, float64 accumulate in feature order (k_docs_embcost's arithmetic).  The
// reference multiplies in float32 while every live track still holds its birth embedding and with BLAS otherwise; both
// differ from this sum in the last bits only.
__global__ void __launch_bounds__(256) k_bt_embcost(const BtCfg cfg, BtStream* streams) {
    const BtStream& s = streams[blockIdx.z];
    const int D = min(*s.n_dets, cfg.cap_dets);
    const int T = s.scalars[SC_N_ACTIVE];
    const int r0 = blockIdx.y * EMB_TR, d0 = blockIdx.x * EMB_TD;
    if (r0 >= T || d0 >= D) return;
    __shared__ double sa[EMB_TR][EMB_TK + 1];
    __shared__ float sb[EMB_TD][EMB_TK + 1];
    __shared__ int slot_of[EMB_TR];
    const int F = cfg.feat_dim;
    const int tr = threadIdx.x / EMB_TD, td = threadIdx.x % EMB_TD;
    if (threadIdx.x < EMB_TR) slot_of[threadIdx.x] = r0 + threadIdx.x < T ? s.tracks[r0 + threadIdx.x] : -1;
    __syncthreads();
    double dot = 0.0;
    for (int k0 = 0; k0 < F; k0 += EMB_TK) {
        for (int e = threadIdx.x; e < EMB_TR * EMB_TK; e += blockDim.x) {
            const int r = e / EMB_TK, k = e % EMB_TK;
            const int slot = slot_of[r];
            sa[r][k] = (slot >= 0 && k0 + k < F) ? s.emb[(size_t)slot * F + k0 + k] : 0.0;
        }
        for (int e = threadIdx.x; e < EMB_TD * EMB_TK; e += blockDim.x) {
            const int d = e / EMB_TK, k = e % EMB_TK;
            sb[d][k] = (d0 + d < D && k0 + k < F) ? s.embs[(size_t)(d0 + d) * F + k0 + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < EMB_TK; ++k) dot += (double)sb[td][k] * sa[tr][k];
        __syncthreads();
    }
    const int slot = slot_of[tr];
    if (slot >= 0 && d0 + td < D) s.embq[(size_t)(d0 + td) * cfg.cap_tracks + slot] = dot;
}

__global__ void __launch_bounds__(256) k_bt_frame(const BtCfg cfg, BtStream* streams, int jv_in_smem) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    BtStream s = streams[blockIdx.x];
    s.jv_wide = jv_in_smem >> 1;
    if (jv_in_smem & 1) jv_scratch_to_smem(s, dyn_smem, max(cfg.cap_tracks, cfg.cap_dets));
    bt_frame(cfg, s);
}

// OccluBoost: the BoostTrack phases with lapjv's scratch in shared memory as k_bt_frame, then its own passes
__global__ void __launch_bounds__(256) k_ob_frame(const ObCfg cfg, ObStream* streams, int jv_in_smem) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    ObStream s = streams[blockIdx.x];
    s.b.jv_wide = jv_in_smem >> 1;
    if (jv_in_smem & 1) jv_scratch_to_smem(s.b, dyn_smem, max(cfg.bt.cap_tracks, cfg.bt.cap_dets));
    ob_frame(cfg, s);
}

// SFSORT: lapjv's scratch in shared memory as k_bt_frame (the square problem is cap_tracks + cap_dets wide); the frames
// themselves never reach the device, only each stream's frame size (margins)
__global__ void __launch_bounds__(256) k_sf_frame(const SfCfg cfg, SfStream* streams, int jv_in_smem) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    SfStream s = streams[blockIdx.x];
    s.jv_wide = jv_in_smem >> 1;
    if (jv_in_smem & 1) jv_scratch_to_smem(s, dyn_smem, cfg.cap_tracks + cfg.cap_dets);
    sf_frame(cfg, s);
}

// ordered (stream, detection) crop list built by one warp with ballot compaction
template <typename Keep>
__device__ __forceinline__ int append_crops(const float* dets, int D, int sidx, int cap_dets, CropDesc* crops, int n, Keep keep) {
    const int lane = threadIdx.x & 31;
    for (int d0 = 0; d0 < D; d0 += 32) {
        const int d = d0 + lane;
        const bool p = d < D && keep(dets + d * 6);
        const unsigned m = __ballot_sync(0xffffffffu, p);
        if (p) {
            const float* r = dets + d * 6;
            CropDesc c;
            c.x1 = r[0]; c.y1 = r[1]; c.x2 = r[2]; c.y2 = r[3];
            c.image = sidx;
            c.out_row = sidx * cap_dets + d;
            crops[n + __popc(m & ((1u << lane) - 1u))] = c;
        }
        n += __popc(m);
    }
    return n;
}

// Which detection rows a family embeds.  The STrack family: the first-round detections
__device__ __forceinline__ bool keep_crop(const TrkCfg& cfg, const float* r) { return (double)r[4] > cfg.high_thresh; }
// DeepOCSORT: every detection above det_thresh (deepocsort.py:333-343)
__device__ __forceinline__ bool keep_crop(const DocsCfg& cfg, const float* r) { return r[4] > cfg.det_thresh_f32; }
// BoostTrack: EVERY detection row.  Which rows survive the confidence boosts depends on the track state, so a
// survivor list would put the ReID behind the association; the frame kernel picks the survivors' rows
__device__ __forceinline__ bool keep_crop(const BtCfg&, const float*) { return true; }

// crop list for on-device ReID: one entry per embedded detection, ordered by (stream, detection)
template <typename Cfg, typename St>
__global__ void k_build_crops(const Cfg cfg, St* streams, int n_streams, CropDesc* crops, int* n_crops, int* hint) {
    if (threadIdx.x >= 32 || blockIdx.x != 0) return;
    int n = 0;
    for (int sidx = 0; sidx < n_streams; ++sidx) {
        const St& s = streams[sidx];
        n = append_crops(s.dets, min(*s.n_dets, cfg.cap_dets), sidx, cfg.cap_dets, crops, n,
                         [&cfg](const float* r) { return keep_crop(cfg, r); });
    }
    if (threadIdx.x == 0) { *n_crops = n; if (hint) *hint = n; }   // hint: host-mapped, read without synchronisation
}

__global__ void k_reset_streams(TrkStream* streams, size_t persistent_bytes) {
    // zero the persistent region of one stream (scalars first, so every list is empty and ids restart at 1)
    TrkStream& s = streams[blockIdx.x];
    uint8_t* base = reinterpret_cast<uint8_t*>(s.scalars);
    for (size_t i = threadIdx.x * 16ull; i < persistent_bytes; i += blockDim.x * 16ull)
        *reinterpret_cast<uint4*>(base + i) = make_uint4(0, 0, 0, 0);
}

// ---------------------------------------------------------------------------------------------------
// Engine
// ---------------------------------------------------------------------------------------------------
static TrkCfg make_core_cfg(const BoxMOTB200TrackerConfig& p) {
    TrkCfg c{};
    const bool bot = p.tracker == BOXMOT_B200_TRACKER_BOTSORT;
    c.kind = bot ? KIND_XYWH : KIND_XYAH;
    c.with_reid = bot ? (p.with_reid ? 1 : 0) : 0;
    c.fuse_first = bot ? (p.fuse_first_associate ? 1 : 0) : 1;
    c.proximity_mask = bot ? 1 : 0;
    c.max_time_lost = (int)((double)p.frame_rate / 30.0 * (double)p.track_buffer);
    c.removed_cap = bot ? p.removed_stracks_buffer : 0;
    c.feat_dim = c.with_reid ? p.feat_dim : 0;
    c.cap_tracks = p.cap_tracks;
    c.cap_dets = p.cap_dets;
    c.vote_cls = bot ? 1 : 0;
    c.high_thresh = p.track_high_thresh;
    c.low_thresh = p.track_low_thresh;
    c.new_thresh_f32 = (float)p.new_track_thresh;
    c.match1 = p.match_thresh;
    c.match2 = p.second_match_thresh;
    c.match3 = p.unconfirmed_match_thresh;
    c.proximity = p.proximity_thresh;
    c.appearance = p.appearance_thresh;
    c.unc_emb_scale = p.unconfirmed_emb_scale;
    return c;
}

template <typename St>
static void upload_streams(const std::vector<St>& h, St** dev) {
    CUDA_OK(cudaMalloc(dev, sizeof(St) * h.size()));
    CUDA_OK(cudaMemcpy(*dev, h.data(), sizeof(St) * h.size(), cudaMemcpyHostToDevice));
}

// TrkStream has no embeddings pointer: the STrack family's appearance prep is handed the source with each launch
static void set_embs(TrkStream&, float*) {}
template <typename St> static void set_embs(St& s, float* embs) { s.embs = embs; }

// Point the carved streams `h` at their slices of input set `set` and of the pending warps, and upload them to *dev.
// Set 0 also records where each stream keeps its output rows, scalars and timers.
template <typename St>
void Engine::wire_streams(std::vector<St>& h, int set, St** dev) {
    const size_t CD = cfg.cap_dets, F = cfg.feat_dim > 0 ? cfg.feat_dim : 1;
    for (int i = 0; i < S; ++i) {
        h[i].dets = in[set].dets + (size_t)i * CD * 6;
        h[i].n_dets = in[set].ndets + i;
        set_embs(h[i], cfg.with_reid ? in[set].embs + (size_t)i * CD * F : nullptr);
        h[i].warp = d_warp + (size_t)i * 8;
        if (set == 0) { out_ptr[i] = h[i].out; scalars_ptr[i] = h[i].scalars; timers_ptr[i] = h[i].timers; }
    }
    upload_streams(h, dev);
}

Engine::Engine(const BoxMOTB200TrackerConfig& p) {
    try {
        construct(p);
    } catch (...) {
        release();   // a failed create must not leak streams, events, device / pinned buffers or ReID models
        throw;
    }
}

void Engine::construct(const BoxMOTB200TrackerConfig& p) {
    if (p.n_streams < 1) throw std::runtime_error("n_streams must be >= 1");
    if (p.cap_tracks < 8 || p.cap_dets < 1) throw std::runtime_error("cap_tracks >= 8 and cap_dets >= 1 required");
    switch (p.tracker) {
        case BOXMOT_B200_TRACKER_BOTSORT:
        case BOXMOT_B200_TRACKER_BYTETRACK: family = Family::STrack; break;
        case BOXMOT_B200_TRACKER_DEEPOCSORT: family = Family::Docs; break;
        case BOXMOT_B200_TRACKER_STRONGSORT: family = Family::StrongSort; break;
        case BOXMOT_B200_TRACKER_BOOSTTRACK: family = Family::Boost; break;
        case BOXMOT_B200_TRACKER_OCCLUBOOST: family = Family::Occlu; break;
        case BOXMOT_B200_TRACKER_SFSORT: family = Family::SfSort; break;
        default: throw std::runtime_error("unknown tracker kind");
    }
    if (p.tracker == BOXMOT_B200_TRACKER_BOTSORT && p.removed_stracks_buffer < 1)
        throw std::runtime_error("removed_stracks_buffer must be >= 1");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        throw std::runtime_error("no CUDA device: boxmot_b200 has no CPU fallback");
    cfg = make_core_cfg(p);
    if (family == Family::Docs) {
        if (p.delta_t < 1 || p.delta_t >= DOCS_RING) throw std::runtime_error("delta_t must be in [1, 7]");
        if (p.max_age < 1 || p.max_age > 46) throw std::runtime_error("max_age must be in [1, 46] (reference history window)");
        dcfg.cap_tracks = p.cap_tracks; dcfg.cap_dets = p.cap_dets; dcfg.feat_dim = p.feat_dim;
        dcfg.delta_t = p.delta_t; dcfg.max_age = p.max_age; dcfg.min_hits = p.min_hits;
        dcfg.embedding_off = p.embedding_off ? 1 : 0; dcfg.aw_off = p.aw_off ? 1 : 0;
        dcfg.det_thresh_f32 = (float)p.det_thresh; dcfg.det_thresh = p.det_thresh;
        dcfg.iou_threshold = p.iou_threshold; dcfg.inertia = p.inertia; dcfg.w_emb = p.w_association_emb;
        dcfg.alpha_fixed = p.alpha_fixed_emb; dcfg.aw_param = p.aw_param; dcfg.q_xy = p.q_xy_scaling; dcfg.q_s = p.q_s_scaling;
        // the shared staging code below reads these from the STrack-family config
        cfg.with_reid = dcfg.embedding_off ? 0 : 1;
        cfg.feat_dim = cfg.with_reid ? p.feat_dim : 0;
        cfg.cap_tracks = p.cap_tracks; cfg.cap_dets = p.cap_dets;
    }
    if (family == Family::StrongSort) {
        if (p.n_init < 1) throw std::runtime_error("n_init must be >= 1");
        if (p.nn_budget < 1) throw std::runtime_error("nn_budget must be >= 1 (the reference's None = unbounded is not supported)");
        if (p.max_age < 1) throw std::runtime_error("max_age must be >= 1");
        scfg.cap_tracks = p.cap_tracks; scfg.cap_dets = p.cap_dets; scfg.feat_dim = p.feat_dim;
        scfg.n_init = p.n_init; scfg.max_age = p.max_age; scfg.budget = p.nn_budget;
        scfg.min_conf = p.min_conf; scfg.max_cos_dist = p.max_cos_dist; scfg.max_iou_dist = p.max_iou_dist;
        scfg.mc_lambda = p.mc_lambda; scfg.ema_alpha = p.ema_alpha;
        cfg.with_reid = 1;   // StrongSORT always associates on appearance
        cfg.feat_dim = p.feat_dim;
        cfg.cap_tracks = p.cap_tracks; cfg.cap_dets = p.cap_dets;
    }
    if (on_bt_stream()) {
        if (p.max_age < 0 || p.max_age > 100000) throw std::runtime_error("max_age must be in [0, 100000]");
        if (p.min_hits < 0) throw std::runtime_error("min_hits must be >= 0");
        btcfg.cap_tracks = p.cap_tracks; btcfg.cap_dets = p.cap_dets;
        btcfg.max_age = p.max_age; btcfg.min_hits = p.min_hits; btcfg.with_reid = p.with_reid ? 1 : 0;
        btcfg.use_dlo = p.use_dlo_boost ? 1 : 0; btcfg.use_duo = p.use_duo_boost ? 1 : 0;
        btcfg.rich_s = p.use_rich_s ? 1 : 0; btcfg.use_sb = p.use_sb ? 1 : 0; btcfg.use_vt = p.use_vt ? 1 : 0;
        btcfg.s_sim_corr = p.s_sim_corr ? 1 : 0;
        btcfg.det_thresh = p.det_thresh; btcfg.iou_threshold = p.iou_threshold;
        btcfg.lambda_iou = p.lambda_iou; btcfg.lambda_mhd = p.lambda_mhd; btcfg.lambda_shape = p.lambda_shape;
        btcfg.dlo_coef = p.dlo_boost_coef; btcfg.min_box_area = p.min_box_area; btcfg.ar_thresh = p.aspect_ratio_thresh;
        cfg.with_reid = btcfg.with_reid;
        cfg.feat_dim = cfg.with_reid ? p.feat_dim : 0;
        cfg.cap_tracks = p.cap_tracks; cfg.cap_dets = p.cap_dets;
    }
    if (family == Family::SfSort) {
        if (p.reid_model_path && p.reid_model_path[0]) throw std::runtime_error("SFSORT has no ReID: pass no ReID blob");
        // the constructor's _resolve_or_default clamps (sfsort.py:205-237)
        auto clamp = [](double v, double lo, double hi) { const double m = hi < v ? hi : v; return m > lo ? m : lo; };
        SfCfg& c = sfcfg;
        c.cap_tracks = p.cap_tracks; c.cap_dets = p.cap_dets;
        c.high_th = clamp(p.sf_high_th, 0.0, 1.0);
        c.match_th_first = clamp(p.sf_match_th_first, 0.0, 0.67);
        c.new_track_th = clamp(p.sf_new_track_th, c.high_th, 1.0);
        c.low_th = clamp(p.sf_low_th, 0.0, c.high_th);
        c.match_th_second = clamp(p.sf_match_th_second, 0.0, 1.0);
        c.cth = clamp(p.sf_cth, c.low_th, 1.0);
        c.dynamic = c.hth_f64 = c.nth_f64 = p.sf_dynamic_tuning ? 1 : 0;   // the tuned thresholds are np.float64
        c.high_th_m = c.dynamic ? clamp(p.sf_high_th_m, 0.02, 0.1) : p.sf_high_th_m;
        c.new_track_th_m = c.dynamic ? clamp(p.sf_new_track_th_m, 0.02, 0.08) : p.sf_new_track_th_m;
        c.match_th_first_m = c.dynamic ? clamp(p.sf_match_th_first_m, 0.02, 0.08) : p.sf_match_th_first_m;
        c.marginal_timeout = (int)clamp(p.sf_marginal_timeout, 0, 500);
        c.central_timeout = (int)clamp(p.sf_central_timeout, 0, 1000);
        c.h_margin = p.sf_horizontal_margin; c.v_margin = p.sf_vertical_margin;
        c.margins_given = p.sf_frame_width > 0 && p.sf_frame_height > 0;
        if (c.margins_given) {
            const double W = p.sf_frame_width, H = p.sf_frame_height;
            c.margin[0] = (float)clamp(c.h_margin, 0.0, W); c.margin[1] = (float)clamp(W - c.h_margin, 0.0, W);
            c.margin[2] = (float)clamp(c.v_margin, 0.0, H); c.margin[3] = (float)clamp(H - c.v_margin, 0.0, H);
        }
        cfg.with_reid = 0;
        cfg.feat_dim = 0;
        cfg.cap_tracks = p.cap_tracks; cfg.cap_dets = p.cap_dets;
    }
    if (cfg.with_reid && cfg.feat_dim < 1) throw std::runtime_error("feat_dim must be set when with_reid");
    S = p.n_streams;
    CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    if (p.reid_model_path && p.reid_model_path[0]) {
        reid = reid_load(p.reid_model_path);
        reid_set_preprocess(reid, p.reid_preprocess);
        if (cfg.with_reid && reid_feature_dim(reid) != cfg.feat_dim) {
            cfg.feat_dim = reid_feature_dim(reid);
        }
    }
    if (family == Family::Docs) dcfg.feat_dim = cfg.feat_dim;
    if (on_bt_stream()) btcfg.feat_dim = cfg.feat_dim;
    if (family == Family::Occlu) {
        if (p.confirm_hits < 1 || p.tentative_max_age < 0 || p.ams_buffer_size < 2 || p.ams_buffer_size > 4096 ||
            p.gta_min_track_length < 1 || p.gta_max_gap < 1)
            throw std::runtime_error("OccluBoost needs confirm_hits >= 1, tentative_max_age >= 0, ams_buffer_size in "
                                     "[2, 4096], gta_min_track_length >= 1 and gta_max_gap >= 1");
        obcfg.bt = btcfg;
        obcfg.use_second_pass = p.use_second_pass ? 1 : 0;
        obcfg.recovery_max_age = p.recovery_max_age; obcfg.second_pass_max_age = p.second_pass_max_age;
        obcfg.second_pass_min_hits = p.second_pass_min_hits; obcfg.confirm_hits = p.confirm_hits;
        obcfg.tentative_max_age = p.tentative_max_age;
        obcfg.ams_on = p.ams_enabled && p.ams_alpha0 < 1.0;   // occluboost.py:791: alpha0 >= 1 never damps nor records
        obcfg.ams_buffer_size = p.ams_buffer_size;
        obcfg.gta = p.gta_enabled && btcfg.with_reid;
        obcfg.gta_min_track_length = p.gta_min_track_length; obcfg.gta_max_gap = p.gta_max_gap;
        obcfg.lambda_emb_mult = p.lambda_emb_multiplier;
        obcfg.recovery_appearance_thresh = p.recovery_appearance_thresh; obcfg.recovery_iou_thresh = p.recovery_iou_thresh;
        obcfg.feat_alpha = p.feat_alpha; obcfg.track_low_thresh = p.track_low_thresh;
        obcfg.second_iou_thresh = p.second_iou_thresh; obcfg.second_appearance_thresh = p.second_appearance_thresh;
        obcfg.new_track_thresh = p.new_track_thresh; obcfg.instant_confirm_thresh = p.instant_confirm_thresh;
        obcfg.duplicate_iou_thresh = p.duplicate_iou_thresh; obcfg.ams_alpha0 = p.ams_alpha0;
        obcfg.ams_threshold = p.ams_threshold; obcfg.ams_shrink_ratio = p.ams_shrink_ratio;
        obcfg.gta_appearance_thresh = p.gta_appearance_thresh;
    }
    if (family == Family::StrongSort) {
        scfg.feat_dim = cfg.feat_dim;
        if (scfg.feat_dim % 4) throw std::runtime_error("StrongSORT feat_dim must be a multiple of 4");
    }
    // every stream's slab of d_mem and the host copy of the struct carved out of it
    auto carve_all = [&](auto carve, const auto& c, auto& h) {
        stream_bytes = carve(c, nullptr, nullptr, &persistent_bytes);
        CUDA_OK(cudaMalloc(&d_mem, stream_bytes * S));
        CUDA_OK(cudaMemset(d_mem, 0, stream_bytes * S));
        h.resize(S);
        for (int i = 0; i < S; ++i) carve(c, d_mem + stream_bytes * i, &h[i], nullptr);
    };
    switch (family) {
        case Family::STrack: carve_all(carve_stream, cfg, h_streams); break;
        case Family::Docs: carve_all(carve_docs, dcfg, h_docs); break;
        case Family::StrongSort: carve_all(carve_ss, scfg, h_ss); break;
        case Family::Boost: carve_all(carve_bt, btcfg, h_bt); break;
        case Family::Occlu:   // its BoostTrack part is what gets wired below; it is put back before the upload
            carve_all(carve_ob, obcfg, h_ob);
            for (const ObStream& o : h_ob) h_bt.push_back(o.b);
            break;
        case Family::SfSort: carve_all(carve_sf, sfcfg, h_sf); break;
    }
    persistent_bytes = (persistent_bytes + 15) & ~(size_t)15;
    const size_t CD = cfg.cap_dets, F = cfg.feat_dim > 0 ? cfg.feat_dim : 1;
    CUDA_OK(cudaMalloc(&in[0].dets, sizeof(float) * 6 * CD * S));
    CUDA_OK(cudaMalloc(&d_warp, sizeof(double) * 8 * S));
    CUDA_OK(cudaMemset(d_warp, 0, sizeof(double) * 8 * S));
    CUDA_OK(cudaMalloc(&in[0].ndets, sizeof(int) * S));
    CUDA_OK(cudaMemset(in[0].ndets, 0, sizeof(int) * S));
    if (cfg.with_reid) {
        CUDA_OK(cudaMalloc(&in[0].embs, sizeof(float) * F * CD * S));
        CUDA_OK(cudaMemset(in[0].embs, 0, sizeof(float) * F * CD * S));
    }
    CUDA_OK(cudaMallocHost(&h_dets, sizeof(float) * 6 * CD * S));
    CUDA_OK(cudaMallocHost(&h_ndets, sizeof(int) * S));
    CUDA_OK(cudaMallocHost(&h_out, sizeof(float) * 8 * CD * S));
    CUDA_OK(cudaMallocHost(&h_scalars, sizeof(int) * SC_COUNT * S));
    if (cfg.with_reid) CUDA_OK(cudaMallocHost(&h_embs, sizeof(float) * F * CD * S));
    CUDA_OK(cudaMalloc(&d_out, sizeof(float) * 8 * CD * S));
    CUDA_OK(cudaMalloc(&d_scalars_out, sizeof(int) * SC_COUNT * S));
    out_ptr.resize(S); scalars_ptr.resize(S); timers_ptr.resize(S);
    if (on_bt_stream()) {
        // KalmanBoxTracker.get_confidence: 0.9 ** k with the host's pow, which is what python's float power calls
        std::vector<double> pw((size_t)(p.max_age + 2 > 8 ? p.max_age + 2 : 8));
        for (size_t k = 0; k < pw.size(); ++k) pw[k] = pow(0.9, (double)k);
        CUDA_OK(cudaMalloc(&d_conf_pow, sizeof(double) * pw.size()));
        CUDA_OK(cudaMemcpy(d_conf_pow, pw.data(), sizeof(double) * pw.size(), cudaMemcpyHostToDevice));
        btcfg.conf_pow = d_conf_pow;
        btcfg.n_conf_pow = (int)pw.size();
        obcfg.bt = btcfg;   // again: the copy taken with the OccluBoost parameters above predates conf_pow
    }
    if (family == Family::SfSort) {
        std::vector<double> lg((size_t)p.cap_dets + 1);
        if (p.sf_log10_table) {
            if (p.sf_log10_count < p.cap_dets + 1) throw std::runtime_error("sf_log10_table needs cap_dets + 1 entries");
            lg.assign(p.sf_log10_table, p.sf_log10_table + lg.size());
        } else {
            sf_log10_table((int)lg.size(), lg.data());
        }
        CUDA_OK(cudaMalloc(&d_log10, sizeof(double) * lg.size()));
        CUDA_OK(cudaMemcpy(d_log10, lg.data(), sizeof(double) * lg.size(), cudaMemcpyHostToDevice));
        sfcfg.log10_tab = d_log10;
        sfcfg.n_log10 = (int)lg.size();
        h_frame_hw.assign((size_t)S * 2, 0);
        CUDA_OK(cudaMalloc(&d_frame_hw, sizeof(int) * 2 * S));
        CUDA_OK(cudaMemset(d_frame_hw, 0, sizeof(int) * 2 * S));
        for (int i = 0; i < S; ++i) h_sf[i].frame_hw = d_frame_hw + 2 * i;
    }
    const bool two_sets = reid && cfg.with_reid;   // second input set for the frame pipeline of update_device
    if (two_sets) {
        CUDA_OK(cudaStreamCreateWithFlags(&reid_stream, cudaStreamNonBlocking));
        CUDA_OK(cudaMalloc(&in[1].dets, sizeof(float) * 6 * CD * S));
        CUDA_OK(cudaMalloc(&in[1].ndets, sizeof(int) * S));
        CUDA_OK(cudaMemset(in[1].ndets, 0, sizeof(int) * S));
        CUDA_OK(cudaMalloc(&in[1].embs, sizeof(float) * F * CD * S));
        CUDA_OK(cudaMemset(in[1].embs, 0, sizeof(float) * F * CD * S));
        for (int k = 0; k < 2; ++k) {
            CUDA_OK(cudaEventCreateWithFlags(&ev_reid_done[k], cudaEventDisableTiming));
            CUDA_OK(cudaEventCreateWithFlags(&ev_assoc_done[k], cudaEventDisableTiming));
        }
    }
    for (int set = two_sets ? 1 : 0; set >= 0; --set) {   // set 0 last: the host copies stay pointed at it
        switch (family) {
            case Family::STrack: wire_streams(h_streams, set, &in[set].trk); break;
            case Family::Docs: wire_streams(h_docs, set, &in[set].docs); break;
            case Family::StrongSort: wire_streams(h_ss, set, &in[set].ss); break;
            case Family::Boost: wire_streams(h_bt, set, &in[set].bt); break;
            case Family::Occlu:
                wire_streams(h_bt, set, &in[set].bt);
                for (int i = 0; i < S; ++i) h_ob[i].b = h_bt[i];
                upload_streams(h_ob, &in[set].ob);
                break;
            case Family::SfSort: wire_streams(h_sf, set, &in[set].sf); break;
        }
    }
    if (reid) {
        CUDA_OK(cudaMalloc(&d_crops, sizeof(CropDesc) * CD * S));
        CUDA_OK(cudaMalloc(&d_ncrops, sizeof(int)));
        // crop count of the most recent frame, written by the crop-list kernel into mapped host memory and read by
        // the host WITHOUT synchronisation: only a balancing hint for the slices (a stale value is still correct)
        CUDA_OK(cudaHostAlloc(&h_crops_hint, sizeof(int), cudaHostAllocMapped));
        *h_crops_hint = 0;
        CUDA_OK(cudaHostGetDevicePointer(&d_crops_hint, h_crops_hint, 0));
        // one H100 80GB HBM3, bench.py default workload (value / e2e frames/s, two runs each): 1 slice 454 / 307-315,
        // 2: 503 / 347, 3: 496 / 334-338, 4: 498-500 / 339-351
        n_split = 2;
        if (const char* sp = getenv("BOXMOT_B200_REID_SPLIT")) n_split = atoi(sp);
        n_split = n_split < 1 ? 1 : (n_split > MAX_SPLIT ? MAX_SPLIT : n_split);
        if (n_split > 1) CUDA_OK(cudaEventCreateWithFlags(&ev_crops, cudaEventDisableTiming));
        for (int k = 0; k + 1 < n_split; ++k) {
            reid_extra[k] = reid_load(p.reid_model_path);
            reid_set_preprocess(reid_extra[k], p.reid_preprocess);
            CUDA_OK(cudaStreamCreateWithFlags(&split_stream[k], cudaStreamNonBlocking));
            CUDA_OK(cudaEventCreateWithFlags(&ev_slice_done[k], cudaEventDisableTiming));
        }
    }
    CUDA_OK(cudaMallocHost(&h_ndets_ring, sizeof(int) * S * NDETS_RING));
    CUDA_OK(cudaEventCreate(&mark[0]));
    CUDA_OK(cudaEventCreate(&mark[1]));
    CUDA_OK(cudaEventCreate(&ev[0]));
    CUDA_OK(cudaEventCreate(&ev[1]));
    CUDA_OK(cudaEventCreate(&ev[2]));
    CUDA_OK(cudaStreamSynchronize(stream));
}

Engine::~Engine() { release(); }

// Everything the constructor acquires; safe on a partially constructed object (members start null).
void Engine::release() {
    if (stream) cudaStreamSynchronize(stream);
    for (int k = 0; k + 1 < n_split; ++k) {
        if (split_stream[k]) { cudaStreamSynchronize(split_stream[k]); cudaStreamDestroy(split_stream[k]); }
        if (ev_slice_done[k]) cudaEventDestroy(ev_slice_done[k]);
        if (reid_extra[k]) reid_free(reid_extra[k]);
    }
    if (ev_crops) cudaEventDestroy(ev_crops);
    if (h_crops_hint) cudaFreeHost(h_crops_hint);
    if (reid_stream) {
        cudaStreamSynchronize(reid_stream);
        cudaStreamDestroy(reid_stream);
        for (int k = 0; k < 2; ++k) {
            if (ev_reid_done[k]) cudaEventDestroy(ev_reid_done[k]);
            if (ev_assoc_done[k]) cudaEventDestroy(ev_assoc_done[k]);
        }
    }
    if (reid) reid_free(reid);
    cudaFree(d_cmc_prev); cudaFree(d_cmc_cur); cudaFree(d_cmc_has_prev); cudaFree(d_cmc_gate);
    if (sof) sof_state_free(sof);
    for (InputSet& s : in) {
        cudaFree(s.dets); cudaFree(s.ndets); cudaFree(s.embs);
        cudaFree(s.trk); cudaFree(s.docs); cudaFree(s.ss); cudaFree(s.bt); cudaFree(s.ob); cudaFree(s.sf);
    }
    cudaFree(d_warp); cudaFree(d_mem); cudaFree(d_out); cudaFree(d_scalars_out); cudaFree(d_conf_pow); cudaFree(d_log10);
    cudaFree(d_frame_hw);
    cudaFree(d_crops); cudaFree(d_ncrops); cudaFree(d_images);
    cudaFreeHost(h_dets); cudaFreeHost(h_ndets); cudaFreeHost(h_out); cudaFreeHost(h_scalars);
    cudaFreeHost(h_embs); cudaFreeHost(h_images); cudaFreeHost(h_ndets_ring);
    if (mark[0]) cudaEventDestroy(mark[0]);
    if (mark[1]) cudaEventDestroy(mark[1]);
    for (auto& e : ev)
        if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
}

void Engine::reset() {
    if (reid_stream) CUDA_OK(cudaStreamSynchronize(reid_stream));
    if (d_cmc_has_prev) CUDA_OK(cudaMemsetAsync(d_cmc_has_prev, 0, sizeof(int) * S, stream));   // ECC.prev_img = None
    if (sof) sof_state_reset(sof, stream);   // a fresh SOF: the next frame initialises
    if (family != Family::STrack) {
        CUDA_OK(cudaStreamSynchronize(stream));
        for (int i = 0; i < S; ++i) CUDA_OK(cudaMemsetAsync(d_mem + stream_bytes * i, 0, persistent_bytes, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        return;
    }
    k_reset_streams<<<S, 256, 0, stream>>>(in[0].trk, persistent_bytes);
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaStreamSynchronize(stream));
}

void Engine::ensure_images(int rows, int cols, bool host_too) {
    size_t need = (size_t)rows * cols * 3;
    if (need > image_bytes) {
        cudaFree(d_images); d_images = nullptr;
        cudaFreeHost(h_images); h_images = nullptr;
        CUDA_OK(cudaMalloc(&d_images, need * S));
        image_bytes = need;
    }
    if (host_too && !h_images) CUDA_OK(cudaMallocHost(&h_images, image_bytes * S));
}

// Enqueue the device work of one frame.  Inputs already in input set 0 (+ embs or images).
void Engine::enqueue_frame(const float* embs_dev, const uint8_t* images_dev, int rows, int cols, int max_dets_total) {
    launches = 0;
    CUDA_OK(cudaEventRecord(ev[0], stream));
    ev_recorded = true;
    if (cmc_mode) enqueue_cmc(images_dev, rows, cols);
    if (cfg.with_reid && !embs_dev) {
        if (!reid)
            throw std::runtime_error(family == Family::StrongSort ? "StrongSORT needs embeddings or a ReID model"
                                     : family == Family::Docs     ? "DeepOCSORT needs embeddings, a ReID model, or embedding_off"
                                     : on_bt_stream()             ? "BoostTrack with_reid needs embeddings or a ReID model"
                                                                  : "with_reid tracker needs embeddings or a ReID model");
        if (!images_dev) throw std::runtime_error("ReID inside update() needs an image");
        enqueue_crops(0, stream);
        launches += run_reid(stream, images_dev, rows, cols, max_dets_total, in[0].embs);
    } else if (cfg.with_reid && family != Family::STrack && embs_dev != in[0].embs) {
        // caller-supplied device embeddings (update_device / DeviceFrameLoop): these families' kernels read the engine's
        // buffer through their stream structs; the STrack family's appearance prep reads the caller's pointer in place
        CUDA_OK(cudaMemcpyAsync(in[0].embs, embs_dev, sizeof(float) * (size_t)cfg.feat_dim * cfg.cap_dets * S,
                                cudaMemcpyDeviceToDevice, stream));
    }
    CUDA_OK(cudaEventRecord(ev[1], stream));
    if (family == Family::SfSort && rows > 0 && cols > 0)   // a frame size given with the batch holds for every stream
        for (int i = 0; i < S; ++i) set_frame_size(i, rows, cols);
    enqueue_family_association(0, embs_dev);
    CUDA_OK(cudaEventRecord(ev[2], stream));
    if (profile) {  // profiling pass: serialise and attribute device time per kernel class
        CUDA_OK(cudaStreamSynchronize(stream));
        float b = 0.f;
        cudaEventElapsedTime(&b, ev[1], ev[2]);
        assoc_ms_accum += b;
        assoc_frames += 1;
    }
}

// crop list of the tracker family from input set `parity`
void Engine::enqueue_crops(int parity, cudaStream_t st) {
    const InputSet& set = in[parity];
    switch (family) {
        case Family::STrack: k_build_crops<<<1, 32, 0, st>>>(cfg, set.trk, S, d_crops, d_ncrops, d_crops_hint); break;
        case Family::Docs: k_build_crops<<<1, 32, 0, st>>>(dcfg, set.docs, S, d_crops, d_ncrops, d_crops_hint); break;
        case Family::StrongSort: ss_build_crops(scfg, set.ss, S, d_crops, d_ncrops, d_crops_hint, st); break;
        case Family::Boost:
        case Family::Occlu: k_build_crops<<<1, 32, 0, st>>>(btcfg, set.bt, S, d_crops, d_ncrops, d_crops_hint); break;
        case Family::SfSort: throw std::runtime_error("SFSORT embeds no detections");
    }
    ++launches;
}

// association launches of the family on `stream`, reading input set `parity` (embeddings included, except that the
// STrack family reads `embs_src` when one is given); a supplied or estimated camera-motion warp applies to this frame only
void Engine::enqueue_family_association(int parity, const float* embs_src) {
    const InputSet& set = in[parity];
    switch (family) {
        case Family::STrack: enqueue_association(set.trk, embs_src ? embs_src : set.embs); break;
        case Family::StrongSort: launches += ss_enqueue_frame(scfg, set.ss, S, stream); break;
        case Family::Boost:
        case Family::Occlu: enqueue_bt(set.bt, set.ob); break;
        case Family::Docs: {
            if (cfg.with_reid) {
                dim3 g((dcfg.cap_dets + EMB_TD - 1) / EMB_TD, (dcfg.cap_tracks + EMB_TR - 1) / EMB_TR, S);
                k_docs_embcost<<<g, 256, 0, stream>>>(dcfg, set.docs);
                ++launches;
            }
            size_t smem;
            const int jv_arg = jv_launch_setup(k_docs_frame, dcfg.cap_tracks, dcfg.cap_dets, &smem);
            k_docs_frame<<<S, 256, smem, stream>>>(dcfg, set.docs, jv_arg);
            ++launches;
            break;
        }
        case Family::SfSort: {
            size_t smem;
            const int jv_arg = jv_launch_setup(k_sf_frame, sfcfg.cap_tracks + sfcfg.cap_dets, 0, &smem);
            k_sf_frame<<<S, 256, smem, stream>>>(sfcfg, set.sf, jv_arg);
            ++launches;
            break;
        }
    }
    if (warp_dirty) {
        CUDA_OK(cudaMemsetAsync(d_warp, 0, sizeof(double) * 8 * S, stream));
        warp_dirty = false;
    }
    CUDA_OK(cudaGetLastError());
}

// BoostTrack / OccluBoost: embedding dot products (wide grid) and the per-stream frame kernel on `stream`
void Engine::enqueue_bt(BtStream* streams_dev, ObStream* ob_dev) {
    BtCfg c = btcfg;
    c.cmc_every_frame = cmc_mode != 0;   // boosttrack.py:318-321: camera_update runs whenever an estimator exists
    if (cfg.with_reid) {
        dim3 g((c.cap_dets + EMB_TD - 1) / EMB_TD, (c.cap_tracks + EMB_TR - 1) / EMB_TR, S);
        k_bt_embcost<<<g, 256, 0, stream>>>(c, streams_dev);
        ++launches;
    }
    size_t smem;
    if (family == Family::Occlu) {
        ObCfg oc = obcfg;
        oc.bt = c;
        const int jv_arg = jv_launch_setup(k_ob_frame, c.cap_tracks, c.cap_dets, &smem);
        k_ob_frame<<<S, 256, smem, stream>>>(oc, ob_dev, jv_arg);
    } else {
        const int jv_arg = jv_launch_setup(k_bt_frame, c.cap_tracks, c.cap_dets, &smem);
        k_bt_frame<<<S, 256, smem, stream>>>(c, streams_dev, jv_arg);
    }
    ++launches;
}

// crop list (already built on main_stream) -> embeddings; slices of the list run concurrently on the helper streams
int Engine::run_reid(cudaStream_t main_stream, const uint8_t* images_dev, int rows, int cols, int total, float* embs_out) {
    const size_t stride = (size_t)rows * cols * 3;
    int n = 0;
    const int ns = (profile || total < 32) ? 1 : n_split;
    if (ns <= 1)
        return reid_forward(reid, images_dev, stride, rows, cols, d_crops, d_ncrops, total, embs_out, cfg.feat_dim, main_stream);
    int expect = *(volatile int*)h_crops_hint;   // crops of a recent frame (0 before the first one)
    if (expect <= 0 || expect > total) expect = total;
    const int per = (((expect + ns - 1) / ns) + 7) & ~7;   // the last slice runs to `total` whatever the hint was
    CUDA_OK(cudaEventRecord(ev_crops, main_stream));
    for (int k = 1; k < ns; ++k) {
        const int a = k * per, b = (k + 1 == ns || (k + 1) * per > total) ? total : (k + 1) * per;
        if (a >= b) continue;
        CUDA_OK(cudaStreamWaitEvent(split_stream[k - 1], ev_crops, 0));
        n += reid_forward(reid_extra[k - 1], images_dev, stride, rows, cols, d_crops, d_ncrops, total, embs_out, cfg.feat_dim,
                          split_stream[k - 1], a, b);
        CUDA_OK(cudaEventRecord(ev_slice_done[k - 1], split_stream[k - 1]));
    }
    n += reid_forward(reid, images_dev, stride, rows, cols, d_crops, d_ncrops, total, embs_out, cfg.feat_dim, main_stream, 0,
                      per < total ? per : total);
    for (int k = 1; k < ns; ++k)
        if (k * per < total) CUDA_OK(cudaStreamWaitEvent(main_stream, ev_slice_done[k - 1], 0));
    return n;
}

// appearance prep + cosine cost (wide grids), the per-stream frame kernel, the deferred appearance EMA: on `stream`
void Engine::enqueue_association(TrkStream* streams_dev, const float* embs_src) {
    if (cfg.with_reid) {
        dim3 g1((cfg.cap_dets + 7) / 8, S);
        k_feat_prepare<<<g1, 256, 0, stream>>>(cfg, streams_dev, embs_src);
        dim3 g2((cfg.cap_dets + EMB_TD - 1) / EMB_TD, (cfg.cap_tracks + EMB_TR - 1) / EMB_TR, S);
        k_embedding_cost<<<g2, 256, 0, stream>>>(cfg, streams_dev);
        launches += 2;
    }
    const size_t lb = lap_smem_bytes(cfg.cap_tracks, cfg.cap_dets);
    const bool in_smem = lb <= 160 * 1024;
    if (in_smem && lb > 48 * 1024)
        CUDA_OK(cudaFuncSetAttribute(k_tracker_frame, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lb));
    k_tracker_frame<<<S, BMB_FRAME_THREADS, in_smem ? lb : 0, stream>>>(cfg, streams_dev, in_smem ? 1 : 0);
    ++launches;
    if (cfg.with_reid) {
        k_feat_ema<<<dim3((cfg.cap_dets + 7) / 8, S), 256, 0, stream>>>(cfg, streams_dev);
        ++launches;
    }
}

// On-device camera-motion estimation: the reference's ECC estimator with its defaults (motion/cmc/ecc.py:23-31), used
// by StrongSORT on every frame that starts with tracks (strongsort.py:67,83-86) and by BoT-SORT with cmc_method "ecc"
// (botsort.py:78,116-117,142).  The estimated warp lands in d_warp like a supplied one and is consumed by the same frame.
void Engine::set_cmc(const char* method) {
    const bool off = !method || !method[0] || strcmp(method, "none") == 0 || strcmp(method, "None") == 0;
    if (off) { cmc_mode = 0; return; }
    if (family == Family::SfSort) throw std::runtime_error("SFSORT has no camera-motion compensation");
    if (strcmp(method, "sof") == 0) {
        // botsort.py:142,301 (every frame, every detection row) and deepocsort.py:330-349 (every frame, the rows with
        // conf > det_thresh); StrongSORT's estimator is ECC
        if (family == Family::StrongSort || is_bytetrack())
            throw std::runtime_error("on-device SOF applies to BoT-SORT and DeepOCSORT (StrongSORT's estimator is ecc)");
        if (!sof) sof = sof_state_create(S, 0.15, 8, 0.2, 3.0);
        else if (cmc_mode != 2) sof_state_reset(sof, stream);
        cmc_mode = 2;
        return;
    }
    if (strcmp(method, "ecc") != 0)
        throw std::runtime_error(std::string("camera-motion method '") + method + "' is not built on the device (ecc, sof, "
                                 "none); orb / sift warps can be supplied through set_warp");
    if (is_bytetrack() || family == Family::Docs)
        throw std::runtime_error("on-device ECC applies to BoT-SORT and StrongSORT (ByteTrack has no CMC, DeepOCSORT's is sof)");
    if (family == Family::StrongSort && !d_cmc_gate) {   // StrongSORT estimates only while tracks exist
        std::vector<const int*> g(S);
        for (int i = 0; i < S; ++i) g[i] = h_ss[i].scalars + SC_N_ACTIVE;
        CUDA_OK(cudaMalloc(&d_cmc_gate, sizeof(const int*) * S));
        CUDA_OK(cudaMemcpy(d_cmc_gate, g.data(), sizeof(const int*) * S, cudaMemcpyHostToDevice));
    }
    cmc_mode = 1;
}

// SFSORT takes a stream's margins from the size of its first frame (BaseTracker._preprocess sets self.w / self.h); the
// frames themselves never reach the device.  Stream-ordered: frames enqueued before the change keep the old size.
void Engine::set_frame_size(int sidx, int rows, int cols) {
    if (family != Family::SfSort) throw std::runtime_error("frame sizes are read by SFSORT handles only");
    if (sidx < 0 || sidx >= S) throw std::runtime_error("stream index out of range");
    if (rows <= 0 || cols <= 0) throw std::runtime_error("frame size must be positive");
    int* hw = h_frame_hw.data() + 2 * sidx;
    if (hw[0] == rows && hw[1] == cols) return;
    hw[0] = rows; hw[1] = cols;
    // pageable source: the copy is staged before the call returns, so h_frame_hw may change afterwards
    CUDA_OK(cudaMemcpyAsync(d_frame_hw + 2 * sidx, hw, sizeof(int) * 2, cudaMemcpyHostToDevice, stream));
}

void Engine::enqueue_cmc(const uint8_t* images_dev, int rows, int cols) {
    if (!images_dev || rows <= 0 || cols <= 0) throw std::runtime_error("camera-motion estimation needs the frame");
    int h, w;
    cmc_scaled_size(rows, cols, cmc_scale, &h, &w);
    if (h < 3 || w < 3) throw std::runtime_error("camera-motion estimation: frame too small for the registration scale");
    if (cmc_mode == 2) {
        const bool docs = family == Family::Docs;
        launches += sof_state_enqueue(sof, images_dev, (size_t)rows * cols * 3, rows, cols, in[0].dets, in[0].ndets,
                                      (int)cfg.cap_dets, 6, docs ? 4 : -1, docs ? dcfg.det_thresh_f32 : 0.f, d_warp, stream);
        warp_dirty = true;   // the estimate applies to this frame only
        return;
    }
    if (h != cmc_h || w != cmc_w) {
        CUDA_OK(cudaStreamSynchronize(stream));
        cudaFree(d_cmc_prev); cudaFree(d_cmc_cur); d_cmc_prev = d_cmc_cur = nullptr;
        CUDA_OK(cudaMalloc(&d_cmc_prev, (size_t)h * w * S));
        CUDA_OK(cudaMalloc(&d_cmc_cur, (size_t)h * w * S));
        if (!d_cmc_has_prev) CUDA_OK(cudaMalloc(&d_cmc_has_prev, sizeof(int) * S));
        CUDA_OK(cudaMemsetAsync(d_cmc_has_prev, 0, sizeof(int) * S, stream));
        cmc_h = h; cmc_w = w;
    }
    cmc_enqueue_ecc(images_dev, (size_t)rows * cols * 3, rows, cols, S, cmc_scale, cmc_eps, cmc_iters, d_cmc_prev, d_cmc_cur,
                    d_cmc_has_prev, d_cmc_gate, d_warp, stream);
    launches += 2;
    warp_dirty = true;   // the estimate applies to this frame only
}

void Engine::set_warp(int sidx, const double* warp6) {
    if (sidx < 0 || sidx >= S) throw std::runtime_error("stream index out of range");
    if (is_bytetrack() || family == Family::SfSort)
        throw std::runtime_error("camera-motion warps apply to BoT-SORT, DeepOCSORT and StrongSORT (ByteTrack and SFSORT have none)");
    double w[8] = {warp6[0], warp6[1], warp6[2], warp6[3], warp6[4], warp6[5], 1.0, 0.0};
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaMemcpy(d_warp + (size_t)sidx * 8, w, sizeof(w), cudaMemcpyHostToDevice));
    warp_dirty = true;
}

void Engine::read_timers(int sidx, long long* out16, bool reset) {
    if (sidx < 0 || sidx >= S) throw std::runtime_error("stream index out of range");
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaMemcpy(out16, timers_ptr[sidx], sizeof(long long) * 16, cudaMemcpyDeviceToHost));
    if (reset) CUDA_OK(cudaMemset(timers_ptr[sidx], 0, sizeof(long long) * 16));
}

void Engine::set_profile(bool on) {
    CUDA_OK(cudaStreamSynchronize(stream));
    profile = on;
    if (reid) reid_set_profile(reid, on);
    assoc_ms_accum = 0.0;
    assoc_frames = 0;
    if (reid) reid_profile_collect(reid, nullptr, nullptr);
}

void Engine::profile_read(double* ms, int* launch_counts) {
    CUDA_OK(cudaStreamSynchronize(stream));
    for (int c = 0; c < REID_N_CLASSES + 1; ++c) { ms[c] = 0.0; launch_counts[c] = 0; }
    if (reid) reid_profile_collect(reid, ms, launch_counts);
    ms[REID_N_CLASSES] = assoc_ms_accum;
    launch_counts[REID_N_CLASSES] = assoc_frames * ((family == Family::Docs || on_bt_stream()) ? (cfg.with_reid ? 2 : 1) : (cfg.with_reid ? 4 : 1));
    assoc_ms_accum = 0.0;
    assoc_frames = 0;
}

void Engine::mark_event(int which) {
    if (which < 0 || which > 1) throw std::runtime_error("mark index must be 0 or 1");
    CUDA_OK(cudaEventRecord(mark[which], stream));
    if (reid_stream && which == 0) CUDA_OK(cudaStreamWaitEvent(reid_stream, mark[0], 0));   // timed region starts here
}

double Engine::marks_elapsed_ms() {
    CUDA_OK(cudaEventSynchronize(mark[1]));
    float t = 0.f;
    CUDA_OK(cudaEventElapsedTime(&t, mark[0], mark[1]));
    return (double)t;
}

void Engine::enqueue_fetch() {
    // gather every stream's rows + scalars into pinned memory (two strided copies)
    CUDA_OK(cudaMemcpy2DAsync(h_out, sizeof(float) * 8 * cfg.cap_dets, out_ptr[0], stream_bytes,
                              sizeof(float) * 8 * cfg.cap_dets, S, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaMemcpy2DAsync(h_scalars, sizeof(int) * SC_COUNT, scalars_ptr[0], stream_bytes,
                              sizeof(int) * SC_COUNT, S, cudaMemcpyDeviceToHost, stream));
}

void Engine::finish_fetch(float* const* out, const int* out_cap, int* out_rows) {
    CUDA_OK(cudaStreamSynchronize(stream));
    for (int i = 0; i < S; ++i) {
        const int* sc = h_scalars + (size_t)i * SC_COUNT;
        if (sc[SC_ERROR] != ERR_NONE) {
            const char* what = sc[SC_ERROR] == ERR_TRACK_CAPACITY ? "track capacity (cap_tracks) exceeded"
                             : sc[SC_ERROR] == ERR_CLS_HIST      ? "more than 8 distinct classes voted on one track"
                             : sc[SC_ERROR] == ERR_LSA_INFEASIBLE ? "assignment cost matrix has no finite solution (NaN / inf costs)"
                                                                 : "detection capacity (cap_dets) exceeded";
            throw std::runtime_error(std::string("stream ") + std::to_string(i) + ": " + what);
        }
        const int m = sc[SC_N_OUT];
        if (out_rows) out_rows[i] = m;
        if (!out || !out[i]) continue;
        if (m > out_cap[i]) throw std::runtime_error("out_capacity_rows too small");
        const float* src = h_out + (size_t)i * cfg.cap_dets * 8;
        for (int r = 0; r < m; ++r) {
            float* o = out[i] + (size_t)r * 9;
            memcpy(o, src + (size_t)r * 8, sizeof(float) * 8);
            o[8] = 0.f;
        }
    }
    if (ev_recorded) {
        float a = 0.f, b = 0.f;
        cudaEventElapsedTime(&a, ev[0], ev[1]);
        cudaEventElapsedTime(&b, ev[1], ev[2]);
        last_reid_ms = a;
        last_assoc_ms = b;
    }
}

void Engine::update_batch(const float* const* dets, const int* det_rows, const float* const* embs,
                          const uint8_t* const* images, int rows, int cols, float* const* out,
                          const int* out_cap, int* out_rows) {
    const size_t CD = cfg.cap_dets, F = cfg.feat_dim > 0 ? cfg.feat_dim : 1;
    int total = 0;
    bool have_embs = cfg.with_reid && embs != nullptr;
    if (reid_stream) CUDA_OK(cudaStreamSynchronize(reid_stream));   // no pipelined frame may still own an input set
    for (int i = 0; i < S; ++i) {
        const int n = det_rows[i];
        if (n < 0 || n > (int)CD) throw std::runtime_error("det_rows exceeds cap_dets");
        h_ndets[i] = n;
        total += n;
        if (n) {
            if (!dets[i]) throw std::runtime_error("dets pointer is NULL");
            memcpy(h_dets + (size_t)i * CD * 6, dets[i], sizeof(float) * 6 * n);
        }
        if (have_embs && n) {
            if (!embs[i]) throw std::runtime_error("embs pointer is NULL for a stream while others pass embeddings");
            memcpy(h_embs + (size_t)i * CD * F, embs[i], sizeof(float) * F * n);
        }
    }
    CUDA_OK(cudaMemcpyAsync(in[0].ndets, h_ndets, sizeof(int) * S, cudaMemcpyHostToDevice, stream));
    // one strided copy moves every stream's occupied prefix; simpler: copy whole staging when small
    for (int i = 0; i < S; ++i) {
        if (!h_ndets[i]) continue;
        CUDA_OK(cudaMemcpyAsync(in[0].dets + (size_t)i * CD * 6, h_dets + (size_t)i * CD * 6,
                                sizeof(float) * 6 * h_ndets[i], cudaMemcpyHostToDevice, stream));
        if (have_embs)
            CUDA_OK(cudaMemcpyAsync(in[0].embs + (size_t)i * CD * F, h_embs + (size_t)i * CD * F,
                                    sizeof(float) * F * h_ndets[i], cudaMemcpyHostToDevice, stream));
    }
    const uint8_t* img_dev = nullptr;
    const bool reid_here = cfg.with_reid && !have_embs;
    if (reid_here || cmc_mode) {
        if (reid_here && !reid) throw std::runtime_error("with_reid tracker needs embeddings or a ReID model");
        if (!images || rows <= 0 || cols <= 0)
            throw std::runtime_error(reid_here ? "ReID inside update() needs an image" : "camera-motion estimation needs the frame");
        ensure_images(rows, cols, true);
        const size_t ib = (size_t)rows * cols * 3;
        for (int i = 0; i < S; ++i) {
            if (!images[i]) throw std::runtime_error("image pointer is NULL");
            // a frame that already lives in page-locked memory goes to the device straight from the caller's
            // buffer (the call returns only after the stream has drained); pageable frames are staged first
            cudaPointerAttributes attr{};
            const bool pinned = cudaPointerGetAttributes(&attr, images[i]) == cudaSuccess && attr.type == cudaMemoryTypeHost;
            if (!pinned) {
                cudaGetLastError();   // unregistered host pointers report an error on some drivers: clear it
                // staged in pieces by a few host threads (host_stage.h); each piece's DMA is queued as soon as it lands
                uint8_t* stage = h_images + ib * i;
                uint8_t* dev = d_images + ib * i;
                StagePool::instance().copy(stage, images[i], ib, [&](size_t off, size_t len) {
                    CUDA_OK(cudaMemcpyAsync(dev + off, stage + off, len, cudaMemcpyHostToDevice, stream));
                });
            } else {
                CUDA_OK(cudaMemcpyAsync(d_images + ib * i, images[i], ib, cudaMemcpyHostToDevice, stream));
            }
        }
        img_dev = d_images;
    }
    enqueue_frame(have_embs ? in[0].embs : nullptr, img_dev, rows, cols, total);
    enqueue_fetch();
    finish_fetch(out, out_cap, out_rows);
}

void Engine::update_device(const float* dets_dev, const int* det_rows, const float* embs_dev,
                           const uint8_t* images_dev, int rows, int cols, bool sync) {
    const size_t CD = cfg.cap_dets;
    int total = 0;
    int* slot = h_ndets_ring + (size_t)(ring_pos++ % NDETS_RING) * S;
    for (int i = 0; i < S; ++i) {
        if (det_rows[i] < 0 || det_rows[i] > (int)CD) throw std::runtime_error("det_rows exceeds cap_dets");
        slot[i] = det_rows[i];
        total += det_rows[i];
    }
    if (can_pipeline() && cfg.with_reid && !embs_dev && images_dev && !sync && !cmc_mode) {
        // frame pipeline: crops + ReID of this frame on reid_stream (input set p), association on `stream` once the
        // embeddings are there; the ReID of the next frame overlaps this frame's association
        const int pp = pipe_parity;
        pipe_parity ^= 1;
        const InputSet& set = in[pp];
        CUDA_OK(cudaStreamWaitEvent(reid_stream, ev_assoc_done[pp], 0));   // set p is free again
        CUDA_OK(cudaMemcpyAsync(set.ndets, slot, sizeof(int) * S, cudaMemcpyHostToDevice, reid_stream));
        if (dets_dev != set.dets)
            CUDA_OK(cudaMemcpyAsync(set.dets, dets_dev, sizeof(float) * 6 * CD * S, cudaMemcpyDeviceToDevice, reid_stream));
        launches = 0;
        ev_recorded = false;   // the per-frame ReID / association split is not timed in pipelined mode
        enqueue_crops(pp, reid_stream);
        launches += run_reid(reid_stream, images_dev, rows, cols, total, set.embs);
        CUDA_OK(cudaEventRecord(ev_reid_done[pp], reid_stream));
        CUDA_OK(cudaStreamWaitEvent(stream, ev_reid_done[pp], 0));
        enqueue_family_association(pp);
        CUDA_OK(cudaEventRecord(ev_assoc_done[pp], stream));
        return;
    }
    if (reid_stream) CUDA_OK(cudaStreamSynchronize(reid_stream));   // leave the pipelined mode in order
    CUDA_OK(cudaMemcpyAsync(in[0].ndets, slot, sizeof(int) * S, cudaMemcpyHostToDevice, stream));
    if (dets_dev != in[0].dets)
        CUDA_OK(cudaMemcpyAsync(in[0].dets, dets_dev, sizeof(float) * 6 * CD * S, cudaMemcpyDeviceToDevice, stream));
    enqueue_frame(cfg.with_reid ? embs_dev : nullptr, images_dev, rows, cols, total);
    if (sync) CUDA_OK(cudaStreamSynchronize(stream));
}

void Engine::fetch(float* const* out, const int* out_cap, int* out_rows) {
    enqueue_fetch();
    finish_fetch(out, out_cap, out_rows);
}

// Where one stream keeps its ordered slot lists and the per-slot identity and Kalman state they index
struct Engine::TrackView {
    const int* scalars;
    int n_lists;                  // list k holds scalars[count[k]] slots
    const int* list[2];
    int count[2];
    const int* id;
    const double* state;          // [cap_tracks][8], the first `dim` used
    const double* cov;            // [cap_tracks][cov_stride], dim x dim row-major
    int dim, cov_stride;
};

Engine::TrackView Engine::track_view(int sidx) const {
    switch (family) {
        case Family::STrack: {
            const TrkStream& s = h_streams[sidx];
            return {s.scalars, 2, {s.active, s.lost}, {SC_N_ACTIVE, SC_N_LOST}, s.id, s.mean, s.cov, 8, 64};
        }
        case Family::StrongSort: {
            const SsStream& s = h_ss[sidx];
            return {s.scalars, 1, {s.tracks, nullptr}, {SC_N_ACTIVE, 0}, s.id, s.mean, s.cov, 8, 64};
        }
        case Family::Docs: {
            const DocsStream& s = h_docs[sidx];
            return {s.scalars, 1, {s.tracks, nullptr}, {SC_N_ACTIVE, 0}, s.id, s.x, s.P, 7, 56};
        }
        case Family::SfSort: {   // no motion state: ids only
            const SfStream& s = h_sf[sidx];
            return {s.scalars, 2, {s.active, s.lost}, {SC_N_ACTIVE, SC_N_LOST}, s.id, nullptr, nullptr, 0, 0};
        }
        default: {
            const BtStream& s = h_bt[sidx];
            return {s.scalars, 1, {s.tracks, nullptr}, {SC_N_ACTIVE, 0}, s.id, s.x, s.P, 8, 64};
        }
    }
}

// Id, state and covariance of every track of the stream's lists in list order, widened to 8 / 8 x 8 with zeros
int Engine::snapshot(int sidx, int* ids, double* means, double* covs, int cap) {
    if (sidx < 0 || sidx >= S) throw std::runtime_error("stream index out of range");
    CUDA_OK(cudaStreamSynchronize(stream));
    const TrackView v = track_view(sidx);
    const int CT = cfg.cap_tracks;
    std::vector<int> sc(SC_COUNT), lst[2], idv(CT);
    std::vector<double> state((size_t)CT * 8), cov((size_t)CT * v.cov_stride);
    CUDA_OK(cudaMemcpy(sc.data(), v.scalars, sizeof(int) * SC_COUNT, cudaMemcpyDeviceToHost));
    for (int l = 0; l < v.n_lists; ++l) {
        lst[l].resize(CT);
        CUDA_OK(cudaMemcpy(lst[l].data(), v.list[l], sizeof(int) * CT, cudaMemcpyDeviceToHost));
    }
    CUDA_OK(cudaMemcpy(idv.data(), v.id, sizeof(int) * CT, cudaMemcpyDeviceToHost));
    if (v.dim) {
        CUDA_OK(cudaMemcpy(state.data(), v.state, sizeof(double) * state.size(), cudaMemcpyDeviceToHost));
        CUDA_OK(cudaMemcpy(cov.data(), v.cov, sizeof(double) * cov.size(), cudaMemcpyDeviceToHost));
    }
    int n = 0;
    for (int l = 0; l < v.n_lists; ++l) {
        for (int k = 0; k < sc[v.count[l]] && n < cap; ++k, ++n) {
            const int t = lst[l][k];
            ids[n] = idv[t];
            for (int i = 0; i < 8; ++i) means[(size_t)n * 8 + i] = i < v.dim ? state[(size_t)t * 8 + i] : 0.0;
            for (int i = 0; i < 64; ++i) covs[(size_t)n * 64 + i] = 0.0;
            for (int i = 0; i < v.dim; ++i)
                for (int j = 0; j < v.dim; ++j) covs[(size_t)n * 64 + i * 8 + j] = cov[(size_t)t * v.cov_stride + i * v.dim + j];
        }
    }
    return n;
}

// OccluBoost resurrection events of one stream (ob_core.cuh), taken and cleared; optionally the graveyard too
int Engine::gta_events(int sidx, int clear_graveyard, double* events, int cap) {
    if (family != Family::Occlu) throw std::runtime_error("GTA events exist on OccluBoost handles only");
    if (sidx < 0 || sidx >= S) throw std::runtime_error("stream index out of range");
    if (reid_stream) CUDA_OK(cudaStreamSynchronize(reid_stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    const ObStream& s = h_ob[sidx];
    int meta[2];
    CUDA_OK(cudaMemcpy(meta, s.gv_meta, sizeof(meta), cudaMemcpyDeviceToHost));
    if (meta[1] > cap) throw std::runtime_error("GTA event buffer too small");
    if (meta[1] > 0) CUDA_OK(cudaMemcpy(events, s.ev, sizeof(double) * OB_EV * meta[1], cudaMemcpyDeviceToHost));
    const int n = meta[1];
    meta[1] = 0;
    if (clear_graveyard) meta[0] = 0;
    CUDA_OK(cudaMemcpy(s.gv_meta, meta, sizeof(meta), cudaMemcpyHostToDevice));
    return n;
}

// Ids of one of the tracker's lists, in list order: 0 = active (the rows `update` may emit), 1 = lost, 2 = removed
// (BaseTracker attributes active_tracks / lost_stracks / removed_stracks, basetracker.py:386-390).  BoT-SORT's removed list
// is its deque(maxlen=removed_stracks_buffer) oldest first; ByteTrack's unbounded list is kept as a per-slot flag, so it
// comes back in slot order.  The other families keep a single list (the reference never fills the other two).
int Engine::track_ids(int sidx, int which, int* ids, int cap) {
    if (sidx < 0 || sidx >= S) throw std::runtime_error("stream index out of range");
    if (which < 0 || which > 2) throw std::runtime_error("list index must be 0 (active), 1 (lost) or 2 (removed)");
    CUDA_OK(cudaStreamSynchronize(stream));
    const TrackView v = track_view(sidx);
    if (which >= v.n_lists && family != Family::STrack) return 0;
    const int CT = cfg.cap_tracks;
    std::vector<int> sc(SC_COUNT), lst(CT), idv(CT);
    int n = 0;
    CUDA_OK(cudaMemcpy(sc.data(), v.scalars, sizeof(int) * SC_COUNT, cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(idv.data(), v.id, sizeof(int) * CT, cudaMemcpyDeviceToHost));
    if (which < v.n_lists) {
        CUDA_OK(cudaMemcpy(lst.data(), v.list[which], sizeof(int) * CT, cudaMemcpyDeviceToHost));
        for (int k = 0; k < sc[v.count[which]] && n < cap; ++k) ids[n++] = idv[lst[k]];
        return n;
    }
    const TrkStream& s = h_streams[sidx];
    if (cfg.removed_cap > 0) {
        std::vector<int> ring(cfg.removed_cap);
        CUDA_OK(cudaMemcpy(ring.data(), s.removed_ring, sizeof(int) * cfg.removed_cap, cudaMemcpyDeviceToHost));
        for (int k = 0; k < sc[SC_RING_COUNT] && n < cap; ++k) ids[n++] = ring[(sc[SC_RING_HEAD] + k) % cfg.removed_cap];
        return n;
    }
    CUDA_OK(cudaMemcpy(lst.data(), s.in_removed, sizeof(int) * CT, cudaMemcpyDeviceToHost));
    for (int t = 0; t < CT && n < cap; ++t)
        if (lst[t]) ids[n++] = idv[t];
    return n;
}

// ---------------------------------------------------------------------------------------------------
// standalone kernels for parity tests / micro-benchmarks
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_lap_only(const TrkCfg cfg, TrkStream* streams, int T, int D, double thresh) {
    TrkStream s = streams[blockIdx.x];
    lap_solve(s, T, D, cfg.cap_dets, thresh);
}

__global__ void __launch_bounds__(256) k_jv_only(DocsStream* streams, int n, int ld, int zrow, int wide) {
    DocsStream s = streams[blockIdx.x];
    jv_dense_solve(s, n, ld, zrow, wide);
}

void set_jv_wide(int mode) { jv_wide_flag() = jv_mode_value(mode); }

// lapjv(cost, extend_cost=True) on an (R, C) float64 host matrix with lapjv's own tie-breaking
void standalone_jv(const double* cost, int R, int C, int* x, int* y) {
    if (R < 0 || C < 0) throw std::runtime_error("negative shape");
    const int n = R > C ? R : C;
    if (n == 0) return;
    DocsCfg c{};
    c.cap_tracks = n < 8 ? 8 : n;
    c.cap_dets = n < 8 ? 8 : n;
    c.feat_dim = 0;
    const int ld = c.cap_tracks;
    size_t bytes = carve_docs(c, nullptr, nullptr, nullptr);
    uint8_t* mem = nullptr;
    DocsStream hs, *ds = nullptr;
    CUDA_OK(cudaMalloc(&mem, bytes));
    CUDA_OK(cudaMemset(mem, 0, bytes));
    carve_docs(c, mem, &hs, nullptr);
    std::vector<double> sq((size_t)n * ld, 0.0);
    for (int i = 0; i < R; ++i)
        for (int j = 0; j < C; ++j) sq[(size_t)i * ld + j] = cost[(size_t)i * C + j];
    CUDA_OK(cudaMalloc(&ds, sizeof(DocsStream)));
    CUDA_OK(cudaMemcpy(ds, &hs, sizeof(DocsStream), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(hs.cost, sq.data(), sizeof(double) * sq.size(), cudaMemcpyHostToDevice));
    k_jv_only<<<1, 256>>>(ds, n, ld, R, jv_wide_default());
    std::vector<int> hx(n), hy(n);
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(hx.data(), hs.lap_x, sizeof(int) * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(hy.data(), hs.lap_y, sizeof(int) * n, cudaMemcpyDeviceToHost);
    cudaFree(mem);
    cudaFree(ds);
    CUDA_OK(e);
    for (int i = 0; i < R; ++i) x[i] = hx[i] < C ? hx[i] : -1;
    for (int j = 0; j < C; ++j) y[j] = hy[j] < R ? hy[j] : -1;
}

void standalone_lap(const double* cost, int T, int D, double thresh, int* x, int* y) {
    if (T < 0 || D < 0) throw std::runtime_error("negative shape");
    if (T == 0 || D == 0) {
        for (int i = 0; i < T; ++i) x[i] = -1;
        for (int j = 0; j < D; ++j) y[j] = -1;
        return;
    }
    TrkCfg c{};
    c.cap_tracks = T < 8 ? 8 : T;
    c.cap_dets = D;
    c.feat_dim = 0;
    size_t bytes = carve_stream(c, nullptr, nullptr, nullptr);
    uint8_t* mem = nullptr;
    TrkStream hs, *ds = nullptr;
    CUDA_OK(cudaMalloc(&mem, bytes));
    CUDA_OK(cudaMemset(mem, 0, bytes));
    carve_stream(c, mem, &hs, nullptr);
    CUDA_OK(cudaMalloc(&ds, sizeof(TrkStream)));
    CUDA_OK(cudaMemcpy(ds, &hs, sizeof(TrkStream), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(hs.cost, cost, sizeof(double) * (size_t)T * D, cudaMemcpyHostToDevice));
    k_lap_only<<<1, 256>>>(c, ds, T, D, thresh);
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(x, hs.lap_x, sizeof(int) * T, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(y, hs.lap_y, sizeof(int) * D, cudaMemcpyDeviceToHost);
    cudaFree(mem);
    cudaFree(ds);
    CUDA_OK(e);
}

__global__ void k_kf_predict(int kind, double* mean, double* cov, const int* tracked, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    TrkCfg c{};
    c.kind = kind;
    kf_predict(c, tracked ? tracked[i] : 1, mean + (size_t)i * 8, cov + (size_t)i * 64);
}
__global__ void k_kf_update(int kind, double* mean, double* cov, const float* meas, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    TrkCfg c{};
    c.kind = kind;
    kf_update(c, meas + (size_t)i * 4, mean + (size_t)i * 8, cov + (size_t)i * 64);
}
__global__ void k_kf_initiate(int kind, const float* meas, double* mean, double* cov, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    TrkCfg c{};
    c.kind = kind;
    kf_initiate(c, meas + (size_t)i * 4, mean + (size_t)i * 8, cov + (size_t)i * 64);
}
__global__ void k_iou_cost(const double* t, int T, const float* d, int D, double* out) {
    size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)T * D) return;
    int i = (int)(e / D), j = (int)(e % D);
    out[e] = iou_dist_td(t + (size_t)i * 4, d + (size_t)j * 4);
}
__global__ void k_cosine_cost(const float* a, int T, const float* b, int D, int F, double* out) {
    size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)T * D) return;
    int i = (int)(e / D), j = (int)(e % D);
    out[e] = cosine_cost_f64(a + (size_t)i * F, b + (size_t)j * F, F);
}

template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    explicit DevBuf(size_t count) : n(count) { if (count) CUDA_OK(cudaMalloc(&p, sizeof(T) * count)); }
    ~DevBuf() { cudaFree(p); }
    void up(const T* h) { if (n) CUDA_OK(cudaMemcpy(p, h, sizeof(T) * n, cudaMemcpyHostToDevice)); }
    void down(T* h) { if (n) CUDA_OK(cudaMemcpy(h, p, sizeof(T) * n, cudaMemcpyDeviceToHost)); }
};

void standalone_kf(int op, int kind, double* mean, double* cov, const int* tracked, const float* meas, int n) {
    if (n <= 0) return;
    DevBuf<double> dm((size_t)n * 8), dc((size_t)n * 64);
    DevBuf<int> dt(tracked ? n : 0);
    DevBuf<float> dz(meas ? (size_t)n * 4 : 0);
    if (op != 2) { dm.up(mean); dc.up(cov); }
    if (tracked) dt.up(tracked);
    if (meas) dz.up(meas);
    int g = (n + 127) / 128;
    if (op == 0) k_kf_predict<<<g, 128>>>(kind, dm.p, dc.p, tracked ? dt.p : nullptr, n);
    else if (op == 1) k_kf_update<<<g, 128>>>(kind, dm.p, dc.p, dz.p, n);
    else k_kf_initiate<<<g, 128>>>(kind, dz.p, dm.p, dc.p, n);
    CUDA_OK(cudaDeviceSynchronize());
    dm.down(mean);
    dc.down(cov);
}

void standalone_iou(const double* t, int T, const float* d, int D, double* out) {
    if (T <= 0 || D <= 0) return;
    DevBuf<double> dt((size_t)T * 4), dout((size_t)T * D);
    DevBuf<float> dd((size_t)D * 4);
    dt.up(t); dd.up(d);
    size_t total = (size_t)T * D;
    k_iou_cost<<<(unsigned)((total + 255) / 256), 256>>>(dt.p, T, dd.p, D, dout.p);
    CUDA_OK(cudaDeviceSynchronize());
    dout.down(out);
}

void standalone_cosine(const float* a, int T, const float* b, int D, int F, double* out) {
    if (T <= 0 || D <= 0) return;
    DevBuf<float> da((size_t)T * F), db((size_t)D * F);
    DevBuf<double> dout((size_t)T * D);
    da.up(a); db.up(b);
    size_t total = (size_t)T * D;
    k_cosine_cost<<<(unsigned)((total + 255) / 256), 256>>>(da.p, T, db.p, D, F, dout.p);
    CUDA_OK(cudaDeviceSynchronize());
    dout.down(out);
}

}  // namespace bmb
