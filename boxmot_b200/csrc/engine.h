// engine.h -- internal C++ interfaces shared by the translation units of libboxmot_b200.so.
#pragma once
#include <cuda_runtime.h>

#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/boxmot_b200.h"
#include "tracker_core.cuh"
#include "docs_core.cuh"
#include "ss_core.cuh"
#include "bt_core.cuh"
#include "ob_core.cuh"
#include "sf_core.cuh"

namespace bmb {

// One detection crop for the ReID path: source frame index, box, and the row of the output matrix it fills.
struct CropDesc {
    float x1, y1, x2, y2;
    int image;
    int out_row;
};

// ---- ReID model (reid_model.cu) -----------------------------------------------------------------------
struct ReidModel;
ReidModel* reid_load(const char* blob_path);  // throws std::runtime_error
void reid_free(ReidModel* m);
int reid_feature_dim(const ReidModel* m);
// crop staging: 0 = resize, 1 = resize_pad (reid/core/preprocessing.py:12-45)
void reid_set_preprocess(ReidModel* m, int mode);
// Enqueue crop -> CNN -> L2-normalised features for up to `max_crops` crops whose descriptors and count live
// in device memory.  Frames are `image_stride` bytes apart in `d_images` (rows x cols x 3, BGR, uint8).
// Row r of the result goes to d_out + crops[r].out_row * out_ld.  Returns the number of kernel launches.
int reid_forward(ReidModel* m, const uint8_t* d_images, size_t image_stride, int rows, int cols,
                 const CropDesc* d_crops, const int* d_ncrops, int max_crops, float* d_out, int out_ld,
                 cudaStream_t stream, int first_crop = 0, int last_crop = -1);
// staged access for the reid C ABI / tests: the normalised input blob (N,256,128,3) float32 NHWC
const float* reid_last_input_blob(const ReidModel* m);
// per-kernel-class device timing: crop, stem, maxpool, pointwise, lightconv, gates, avgpool, head
constexpr int REID_N_CLASSES = 8;
void reid_set_profile(ReidModel* m, bool on);
void reid_profile_collect(ReidModel* m, double* ms, int* launches);
// diagnostics: stop the next forward after stage `stage` (0 blob, 1 stem, 2 pool, 3.. block / transition outputs,
// 11 conv5; -1 = run to the end) and expose that NHWC tensor of the first chunk
void reid_set_debug_stop(ReidModel* m, int stage);
const float* reid_debug_tensor(const ReidModel* m, size_t* floats_per_crop);

struct SofState;   // cmc_sof_kernels.cu

// ---- tracker engine (tracker_engine.cu) -----------------------------------------------------------------
struct Engine {
    TrkCfg cfg{};
    int S = 0;
    cudaStream_t stream = nullptr;
    ReidModel* reid = nullptr;
    uint8_t* d_mem = nullptr;
    size_t stream_bytes = 0, persistent_bytes = 0;
    // Which tracker runs: the STrack family (ByteTrack / BoT-SORT, tracker_core.cuh), DeepOCSORT / OC-SORT (docs_core.cuh),
    // StrongSORT (ss_core.cuh), BoostTrack (bt_core.cuh), OccluBoost (ob_core.cuh, whose streams wrap a BtStream) or
    // SFSORT (sf_core.cuh).
    enum class Family { STrack, Docs, StrongSort, Boost, Occlu, SfSort };
    Family family = Family::STrack;
    bool on_bt_stream() const { return family == Family::Boost || family == Family::Occlu; }
    bool is_bytetrack() const { return family == Family::STrack && cfg.kind != KIND_XYWH; }
    // family configs and host copies of the stream structs of input set 0 (h_bt holds OccluBoost's BoostTrack part too)
    DocsCfg dcfg{};
    SsCfg scfg{};
    BtCfg btcfg{};
    ObCfg obcfg{};
    SfCfg sfcfg{};
    std::vector<TrkStream> h_streams;
    std::vector<DocsStream> h_docs;
    std::vector<SsStream> h_ss;
    std::vector<BtStream> h_bt;
    std::vector<ObStream> h_ob;
    std::vector<SfStream> h_sf;
    // One set of frame inputs and the family's device stream array that reads it.  Set 0 serves update() and the
    // synchronous device path; set 1 exists with on-device ReID, for the frame pipeline of update_device.
    struct InputSet {
        float* dets = nullptr;
        int* ndets = nullptr;
        float* embs = nullptr;
        TrkStream* trk = nullptr;
        DocsStream* docs = nullptr;
        SsStream* ss = nullptr;
        BtStream* bt = nullptr;
        ObStream* ob = nullptr;
        SfStream* sf = nullptr;
    };
    InputSet in[2];
    double* d_conf_pow = nullptr;      // 0.9 ** k, k = 0 .. max_age + 1 (KalmanBoxTracker.get_confidence)
    double* d_log10 = nullptr;         // SFSORT: log10(k), k = 0 .. cap_dets (_dynamic_thresholds)
    int* d_frame_hw = nullptr;         // SFSORT: [S][2] frame size of each stream (its margins come from the first)
    std::vector<int> h_frame_hw;
    std::vector<float*> out_ptr;       // per-stream output rows / scalars / timers (either family)
    std::vector<int*> scalars_ptr;
    std::vector<long long*> timers_ptr;
    double* d_warp = nullptr;      // [S][8] pending camera-motion warps (slot 6 = pending flag)
    bool warp_dirty = false;
    // on-device camera-motion estimation: 0 = off (warps are supplied), 1 = the reference's ECC defaults (cmc_ecc.cuh),
    // 2 = the reference's SOF defaults (cmc_sof.cuh)
    int cmc_mode = 0;
    double cmc_scale = 0.15, cmc_eps = 1e-5;
    int cmc_iters = 100;
    int cmc_h = 0, cmc_w = 0;            // registration image size of the frames seen so far
    uint8_t* d_cmc_prev = nullptr;       // [S][cmc_h * cmc_w] previous registration image per stream
    uint8_t* d_cmc_cur = nullptr;
    int* d_cmc_has_prev = nullptr;       // [S]
    const int** d_cmc_gate = nullptr;    // [S] device pointers to the live-track count (StrongSORT) or null
    SofState* sof = nullptr;             // cmc_mode 2: the reference's SOF estimator (BoT-SORT, DeepOCSORT)
    float* d_out = nullptr;
    int* d_scalars_out = nullptr;
    CropDesc* d_crops = nullptr;
    int* d_ncrops = nullptr;
    uint8_t* d_images = nullptr;
    size_t image_bytes = 0;
    float* h_dets = nullptr;
    int* h_ndets = nullptr;
    float* h_out = nullptr;
    int* h_scalars = nullptr;
    float* h_embs = nullptr;
    uint8_t* h_images = nullptr;
    cudaEvent_t ev[3]{};
    cudaEvent_t mark[2]{};
    int* h_ndets_ring = nullptr;   // pinned ring so that queued frames keep their own det counts
    int ring_pos = 0;
    static constexpr int NDETS_RING = 256;
    double assoc_ms_accum = 0.0;
    int assoc_frames = 0;
    // frame pipeline of the device-resident path (update_device): ReID of frame f+1 runs on its own stream while
    // the single-CTA-per-stream association of frame f runs on `stream`; inputs are double-buffered (in[0] / in[1])
    cudaStream_t reid_stream = nullptr;
    // extra ReID workspaces: slices of a frame's crop list run concurrently on helper streams (the tile kernels
    // are latency-bound with short waves; concurrent slices fill each other's tails)
    static constexpr int MAX_SPLIT = 4;
    int n_split = 1;
    ReidModel* reid_extra[MAX_SPLIT - 1]{};
    cudaStream_t split_stream[MAX_SPLIT - 1]{};
    cudaEvent_t ev_crops = nullptr;
    int* h_crops_hint = nullptr;           // mapped host word: crop count of a recent frame (slice balancing hint)
    int* d_crops_hint = nullptr;
    cudaEvent_t ev_slice_done[MAX_SPLIT - 1]{};
    cudaEvent_t ev_reid_done[2]{};
    cudaEvent_t ev_assoc_done[2]{};
    int pipe_parity = 0;
    bool ev_recorded = false;
    bool profile = false;
    int launches = 0;
    double last_reid_ms = 0.0, last_assoc_ms = 0.0;

    explicit Engine(const BoxMOTB200TrackerConfig& p);
    ~Engine();
    Engine(const Engine&) = delete;
    Engine& operator=(const Engine&) = delete;

    void reset();
    void update_batch(const float* const* dets, const int* det_rows, const float* const* embs,
                      const uint8_t* const* images, int rows, int cols, float* const* out, const int* out_cap,
                      int* out_rows);
    void update_device(const float* dets_dev, const int* det_rows, const float* embs_dev,
                       const uint8_t* images_dev, int rows, int cols, bool sync);
    void fetch(float* const* out, const int* out_cap, int* out_rows);
    int snapshot(int stream_index, int* ids, double* means, double* covs, int cap);
    int track_ids(int stream_index, int which, int* ids, int cap);
    int gta_events(int stream_index, int clear_graveyard, double* events, int cap);
    void set_warp(int stream_index, const double* warp6);
    void set_cmc(const char* method);   // "ecc" | "sof" | "none" / "" / NULL
    void set_frame_size(int stream_index, int rows, int cols);   // SFSORT: the size of the stream's frames
    void read_timers(int stream_index, long long* out16, bool reset);
    void set_profile(bool on);
    void profile_read(double* ms, int* launch_counts);  // REID_N_CLASSES + 1 entries (last = association)
    void mark_event(int which);
    double marks_elapsed_ms();

   private:
    void construct(const BoxMOTB200TrackerConfig& p);
    void release();
    void ensure_images(int rows, int cols, bool host_too);
    void enqueue_cmc(const uint8_t* images_dev, int rows, int cols);
    void enqueue_frame(const float* embs_dev, const uint8_t* images_dev, int rows, int cols, int max_dets_total);
    bool can_pipeline() const { return reid_stream != nullptr && !profile; }
    template <typename St> void wire_streams(std::vector<St>& h, int set, St** dev);
    void enqueue_association(TrkStream* streams_dev, const float* embs_src);
    void enqueue_crops(int parity, cudaStream_t st);            // crop list of the family, from input set `parity`
    // association launches of the family on `stream`; the STrack family reads `embs_src` in place (null: the set's own)
    void enqueue_family_association(int parity, const float* embs_src = nullptr);
    void enqueue_bt(BtStream* streams_dev, ObStream* ob_dev);    // BoostTrack / OccluBoost: embedding cost + frame kernel
    struct TrackView;
    TrackView track_view(int stream_index) const;
    int run_reid(cudaStream_t main_stream, const uint8_t* images_dev, int rows, int cols, int total, float* embs_out);
    void enqueue_fetch();
    void finish_fetch(float* const* out, const int* out_cap, int* out_rows);
};

// ---- StrongSORT kernels (ss_kernels.cu) ---------------------------------------------------------------------
void ss_build_crops(const SsCfg& cfg, SsStream* d_streams, int S, CropDesc* crops, int* n_crops, int* hint,
                    cudaStream_t stream);
// unit detection rows -> gallery distances -> per-stream frame -> appearance / gallery update; returns launches
int ss_enqueue_frame(const SsCfg& cfg, SsStream* d_streams, int S, cudaStream_t stream);
int standalone_lsa(const double* cost, int R, int C, int* row_ind, int* col_ind);

// ---- camera-motion estimation (cmc_kernels.cu) ---------------------------------------------------------------
// dsize of cv2.resize(src, (0, 0), fx=scale, fy=scale): saturate_cast<int>(n * scale), round half to even
inline void cmc_scaled_size(int rows, int cols, double scale, int* h, int* w) {
    *h = (int)nearbyint(rows * scale);
    *w = (int)nearbyint(cols * scale);
}
// BaseCMC.preprocess of S frames (image_stride bytes apart) into out [S][h * w]
void cmc_enqueue_prepare(const uint8_t* images, size_t image_stride, int rows, int cols, int S, double scale, uint8_t* out,
                         cudaStream_t st);
void cmc_enqueue_ecc(const uint8_t* images, size_t image_stride, int rows, int cols, int S, double scale, double eps,
                     int max_iter, uint8_t* prev, uint8_t* cur, int* has_prev, const int* const* gate, double* warp,
                     cudaStream_t st);
void standalone_ecc(const uint8_t* prev_bgr, const uint8_t* cur_bgr, int rows, int cols, double scale, double eps,
                    int max_iter, float* warp6, int* status, uint8_t* prepared_out);

// ---- SOF camera-motion estimator (cmc_sof_kernels.cu) ---------------------------------------------------------------
// SofState: per-stream estimator state of S streams (pyramids, keypoints, workspace sized from the registration image)
SofState* sof_state_create(int S, double scale, int min_inliers, double min_ratio, double ransac_thresh);
void sof_state_free(SofState* st);
void sof_state_reset(SofState* st, cudaStream_t cs);   // every stream initialises again on its next frame
// SOF.apply for S frames (device, image_stride bytes apart); the boxes of the detection rows dets [S][det_cap][det_stride]
// (n: ndets[S]; with conf_col >= 0 only rows with row[conf_col] > conf_thr) leave the corner mask.  Accepted warps land
// in warp8 [S][8] with the pending flag set.  Returns the number of launches.
int sof_state_enqueue(SofState* st, const uint8_t* images, size_t image_stride, int rows, int cols, const float* dets,
                      const int* ndets, int det_cap, int det_stride, int conf_col, float conf_thr, double* warp8,
                      cudaStream_t cs);
// standalone handle (boxmot_b200_cmc_sof_*)
void* sof_create(double scale, int min_inliers, double min_ratio, double ransac_thresh);
void sof_apply(void* handle, const uint8_t* bgr, int rows, int cols, const float* dets_xyxy, int n_dets, float* warp6,
               int* status);
void sof_destroy(void* handle);

void standalone_jv(const double* cost, int R, int C, int* x, int* y);
void set_jv_wide(int mode);   // dense-JV augmentation variant used by every later launch of this process
void standalone_lap(const double* cost, int T, int D, double thresh, int* x, int* y);
void standalone_kf(int op, int kind, double* mean, double* cov, const int* tracked, const float* meas, int n);
void standalone_iou(const double* t, int T, const float* d, int D, double* out);
void standalone_cosine(const float* a, int T, const float* b, int D, int F, double* out);
void standalone_pointwise(const float* A, int M, int K, const float* W, int N, const float* bias, const float* residual,
                          int relu, int use_tc, float* out, float* elapsed_ms);
void standalone_instance_norm(const float* x, int n, int H, int W, int C, const float* gamma, const float* beta,
                              const float* residual, int relu, int pool, float* out);
void standalone_resnet_conv(const float* in0, int n, int h0, int w0, int c0, int k, int stride, const float* in1, int h1,
                            int w1, int c1, int stride1, const float* w, int N, const float* bias, const float* residual,
                            int relu, float* out, float* elapsed_ms);
void standalone_vit_layernorm(const float* x, int rows, const float* gamma, const float* beta, float* out);
void standalone_vit_attention(const float* qkv, int n, int tokens, float* out, int width);
void standalone_vits_layernorm(const float* x, int rows, const float* gamma, const float* beta, float* out);
void standalone_vits_ain(const float* x, int n, int tokens, const float* a, const float* b, const float* s, float* out);
void standalone_vits_head(const float* x, int n, int gh, int gw, int pool, int proj, const float* hw, int n_hw,
                          int normalise, float* out);
void standalone_mlfn_group_conv(const float* in, int n, int h, int w, int c, int gw, int stride, const float* weight,
                                const float* bias, const float* gates, float* out);
void standalone_mlfn_fsm(const float* x, int n, int h, int w, int c, const float* w1, const float* b1, int f0,
                         const float* w2, const float* b2, int f1, const float* w3, const float* b3, float* out);
void standalone_f32_pointwise(const float* a, const float* branches, const float* gates, int n, int hw, int k, int mid,
                              const float* w, int nout, const float* bias, const float* residual, int relu, int off,
                              int count, float* out, int out_floats, int* instance);
void standalone_f32_lightconv(const float* in, int nb, int n, int h, int w, int c, const float* wpw, const float* wdw,
                              const float* bias, int off, int count, float* out, int out_stride, float* sums,
                              int sums_stride, int* instance);
void standalone_f32_lightchain(const float* in, int n, int h, int w, int c, const float* wpw, const float* wdw,
                               const float* bias, int off, int count, float* out, int out_stride, float* sums,
                               int sums_stride, int* instance);
void standalone_f32_gates(const float* sums, int n, int tiles, int c, int hid, int hw, const float* w1, const float* b1,
                          const float* w2, const float* b2, int off, int count, float* gates, int gates_floats);
void standalone_f32_head(const float* x, int n, int hw, int c, const float* wfc, const float* bfc, int feat,
                         const int* rows, int off, int count, float* out, int out_floats, int out_ld);
void standalone_f32_map(int op, const float* in, int n, int h, int w, int c, int stride, const float* weight,
                        const float* bias, int off, int count, float* out, int out_floats);
void standalone_f32_lmbn_head(const float* x, int n, int h, int w, const float* neck, const int* rows, int off,
                              int count, float* pooled, int pooled_floats, float* out, int out_floats, int out_ld);

void standalone_hacnn_conv(const float* in, int n, int off, int count, int h, int w, int c0, int k, int stride,
                           const float* weight, int N, const float* bias, float* out, int out_ld, int out_off);
void standalone_hacnn_map(int op, const float* in, int n, int off, int count, int h, int w, int c, const float* weight,
                          const float* bias, float* out);
void standalone_hacnn_attention(const float* x, int n, int off, int count, int h, int w, int c, int level,
                                const float* params, float* out, float* s, float* v, float* theta);
void standalone_hacnn_stn(const float* src, int n, int off, int count, int H, int W, int C, const float* theta,
                          int level, const float* prev, int lh, int lw, float* out);
void standalone_hacnn_head(const float* x3, int n, int off, int count, int hw3, const float* loc, int hwl,
                           const float* wg, const float* bg, const float* wl, const float* bl, const int* rows,
                           int out_rows, float* out, float* v);

void standalone_cspreid_conv(const float* in, int n, int off, int count, int h, int w, int c0, int in_ld, int in_off,
                             int k, int stride, const float* weight, int N, const float* bias, const float* residual,
                             int res_ld, int res_off, float* out, int out_ld, int out_off);
void standalone_cspreid_map(int op, const float* in, int n, int off, int count, int h, int w, int c,
                            const float* weight, const float* bias, float* out);
void standalone_cspreid_attention(const float* x, int n, int off, int count, int h, int w, const float* params,
                                  float* out);
void standalone_cspreid_head(const float* x, int n, int off, int count, int h, int w, const float* params,
                             const int* rows, int out_rows, float* out, float* raw);

}  // namespace bmb
