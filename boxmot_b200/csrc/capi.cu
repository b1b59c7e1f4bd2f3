// capi.cu -- the extern "C" surface of libboxmot_b200.so (see include/boxmot_b200.h for the contract and the
// reference interfaces each symbol replaces).  Errors never cross the ABI: every entry point is wrapped, the
// message is kept in a thread-local string (native_runtime.hpp:17-29 GuardCall convention).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <stdexcept>
#include <string>
#include <vector>

#include "engine.h"

using namespace bmb;

namespace {
thread_local std::string g_error;

template <typename Fn>
int guard(Fn&& fn) {
    try {
        g_error.clear();
        fn();
        return 1;
    } catch (const std::exception& e) {
        g_error = e.what();
    } catch (...) {
        g_error = "unknown error";
    }
    return 0;
}

bool cmc_requested(const char* m) {
    return m && m[0] && strcmp(m, "none") != 0 && strcmp(m, "None") != 0;
}

void check_update_args(int det_rows, int det_cols, int out_cols, const float* dets, const float* out, int out_cap) {
    if (det_rows < 0) throw std::runtime_error("det_rows < 0");
    if (det_rows > 0 && det_cols == 7)
        throw std::runtime_error("OBB detections (7 columns) are out of scope for the B200 path");
    if (det_rows > 0 && det_cols != 6)
        throw std::runtime_error("Unsupported 'dets' 2nd dimension length, valid length is 6 (x1,y1,x2,y2,conf,cls)");
    if (det_rows > 0 && !dets) throw std::runtime_error("dets is NULL");
    if (out_cols != 9) throw std::runtime_error("out_cols must be 9");
    if (!out || out_cap < 1) throw std::runtime_error("out_tracks / out_capacity_rows invalid");
}

Engine* as_engine(void* h) {
    if (!h) throw std::runtime_error("NULL handle");
    return reinterpret_cast<Engine*>(h);
}

int single_update(void* handle, const float* dets, int det_rows, int det_cols, const float* embs, int emb_rows,
                  int emb_cols, const uint8_t* image, int rows, int cols, int ch, float* out, int out_cap,
                  int out_cols, int* out_rows, int* out_is_obb) {
    return guard([&] {
        Engine* e = as_engine(handle);
        if (e->S != 1) throw std::runtime_error("handle holds several streams: use boxmot_b200_tracker_update_batch");
        check_update_args(det_rows, det_cols, out_cols, dets, out, out_cap);
        if (embs) {
            if (emb_rows != det_rows) throw std::runtime_error("Missmatch between detections and embeddings sizes");
            if (e->cfg.with_reid && det_rows > 0 && emb_cols != e->cfg.feat_dim)
                throw std::runtime_error("embedding width does not match feat_dim");
        }
        if (image && ch != 3 && e->cfg.with_reid && !embs) throw std::runtime_error("image must be HxWx3 uint8 BGR");
        const float* dp[1] = {dets};
        const float* ep[1] = {embs};
        const uint8_t* ip[1] = {image};
        float* op[1] = {out};
        int n = 0;
        e->update_batch(dp, &det_rows, (embs && e->cfg.with_reid) ? ep : nullptr, image ? ip : nullptr, rows, cols,
                        op, &out_cap, &n);
        if (out_rows) *out_rows = n;
        if (out_is_obb) *out_is_obb = 0;
    });
}
}  // namespace

extern "C" {

const char* boxmot_b200_last_error(void) { return g_error.c_str(); }
const char* boxmot_bytetrack_last_error(void) { return g_error.c_str(); }
const char* boxmot_botsort_last_error(void) { return g_error.c_str(); }
const char* boxmot_sfsort_last_error(void) { return g_error.c_str(); }

int boxmot_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// ---- generic tracker ------------------------------------------------------------------------------------
BoxMOTB200Tracker* boxmot_b200_tracker_create(const BoxMOTB200TrackerConfig* config) {
    Engine* e = nullptr;
    guard([&] {
        if (!config) throw std::runtime_error("NULL config");
        e = new Engine(*config);
    });
    return reinterpret_cast<BoxMOTB200Tracker*>(e);
}
void boxmot_b200_tracker_destroy(BoxMOTB200Tracker* h) {
    guard([&] { delete reinterpret_cast<Engine*>(h); });
}
int boxmot_b200_tracker_reset(BoxMOTB200Tracker* h) {
    return guard([&] { as_engine(h)->reset(); });
}
int boxmot_b200_tracker_update_batch(BoxMOTB200Tracker* h, const float* const* dets, const int* det_rows,
                                     const float* const* embs, const uint8_t* const* images, int image_rows,
                                     int image_cols, float* const* out, const int* out_capacity_rows,
                                     int* out_rows) {
    return guard([&] {
        if (!dets || !det_rows || !out || !out_capacity_rows) throw std::runtime_error("NULL argument");
        as_engine(h)->update_batch(dets, det_rows, embs, images, image_rows, image_cols, out, out_capacity_rows,
                                   out_rows);
    });
}
int boxmot_b200_tracker_update_device(BoxMOTB200Tracker* h, const float* d_dets, const int* det_rows,
                                      const float* d_embs, const uint8_t* d_images, int image_rows, int image_cols,
                                      int sync) {
    return guard([&] {
        if (!d_dets || !det_rows) throw std::runtime_error("NULL argument");
        as_engine(h)->update_device(d_dets, det_rows, d_embs, d_images, image_rows, image_cols, sync != 0);
    });
}
int boxmot_b200_tracker_fetch(BoxMOTB200Tracker* h, float* const* out, const int* out_capacity_rows, int* out_rows) {
    return guard([&] { as_engine(h)->fetch(out, out_capacity_rows, out_rows); });
}
int boxmot_b200_tracker_snapshot(BoxMOTB200Tracker* h, int stream, int* ids, double* means, double* covs,
                                 int capacity, int* out_count) {
    return guard([&] {
        int n = as_engine(h)->snapshot(stream, ids, means, covs, capacity);
        if (out_count) *out_count = n;
    });
}
int boxmot_b200_tracker_track_ids(BoxMOTB200Tracker* h, int stream, int which, int* ids, int capacity, int* out_count) {
    return guard([&] {
        int n = as_engine(h)->track_ids(stream, which, ids, capacity);
        if (out_count) *out_count = n;
    });
}
int boxmot_b200_tracker_gta_events(BoxMOTB200Tracker* h, int stream, int clear_graveyard, double* events, int capacity,
                                   int* out_count) {
    return guard([&] {
        int n = as_engine(h)->gta_events(stream, clear_graveyard, events, capacity);
        if (out_count) *out_count = n;
    });
}
int boxmot_b200_tracker_last_launches(BoxMOTB200Tracker* h, int* out_launches) {
    return guard([&] { *out_launches = as_engine(h)->launches; });
}
int boxmot_b200_tracker_last_device_ms(BoxMOTB200Tracker* h, double* reid_ms, double* assoc_ms) {
    return guard([&] {
        Engine* e = as_engine(h);
        if (reid_ms) *reid_ms = e->last_reid_ms;
        if (assoc_ms) *assoc_ms = e->last_assoc_ms;
    });
}

int boxmot_b200_tracker_set_warp(BoxMOTB200Tracker* h, int stream, const double* warp2x3) {
    return guard([&] {
        if (!warp2x3) throw std::runtime_error("warp is NULL");
        as_engine(h)->set_warp(stream, warp2x3);
    });
}
int boxmot_b200_tracker_set_frame_size(BoxMOTB200Tracker* h, int stream, int rows, int cols) {
    return guard([&] { as_engine(h)->set_frame_size(stream, rows, cols); });
}
int boxmot_b200_tracker_set_cmc(BoxMOTB200Tracker* h, const char* method) {
    return guard([&] { as_engine(h)->set_cmc(method); });
}
int boxmot_b200_tracker_mark(BoxMOTB200Tracker* h, int which) {
    return guard([&] { as_engine(h)->mark_event(which); });
}
int boxmot_b200_tracker_elapsed_ms(BoxMOTB200Tracker* h, double* out_ms) {
    return guard([&] { *out_ms = as_engine(h)->marks_elapsed_ms(); });
}
int boxmot_b200_tracker_phase_clocks(BoxMOTB200Tracker* h, int stream, long long* out16, int reset) {
    return guard([&] { as_engine(h)->read_timers(stream, out16, reset != 0); });
}
int boxmot_b200_tracker_profile(BoxMOTB200Tracker* h, int enable) {
    return guard([&] { as_engine(h)->set_profile(enable != 0); });
}
int boxmot_b200_tracker_profile_read(BoxMOTB200Tracker* h, double* ms, int* launches) {
    return guard([&] { as_engine(h)->profile_read(ms, launches); });
}

// ---- ByteTrack (reference ABI) ----------------------------------------------------------------------------
BoxMOTByteTrackHandle* boxmot_bytetrack_create(const BoxMOTByteTrackConfig* c) {
    Engine* e = nullptr;
    guard([&] {
        if (!c) throw std::runtime_error("NULL config");
        BoxMOTB200TrackerConfig p{};
        p.tracker = BOXMOT_B200_TRACKER_BYTETRACK;
        p.n_streams = 1;
        p.cap_tracks = 4096;
        p.cap_dets = 1024;
        p.track_buffer = c->track_buffer;
        p.frame_rate = c->frame_rate;
        p.track_high_thresh = c->track_thresh;
        p.track_low_thresh = c->min_conf;
        p.new_track_thresh = c->track_thresh;
        p.match_thresh = c->match_thresh;
        p.second_match_thresh = 0.5;       // bytetrack.py:336
        p.unconfirmed_match_thresh = 0.7;  // bytetrack.py:358
        e = new Engine(p);
    });
    return reinterpret_cast<BoxMOTByteTrackHandle*>(e);
}
void boxmot_bytetrack_destroy(BoxMOTByteTrackHandle* h) { guard([&] { delete reinterpret_cast<Engine*>(h); }); }
int boxmot_bytetrack_reset(BoxMOTByteTrackHandle* h) { return guard([&] { as_engine(h)->reset(); }); }
int boxmot_bytetrack_update(BoxMOTByteTrackHandle* h, const float* dets, int det_rows, int det_cols,
                            const uint8_t* image, int rows, int cols, int ch, float* out, int out_cap, int out_cols,
                            int* out_rows, int* out_is_obb) {
    return single_update(h, dets, det_rows, det_cols, nullptr, 0, 0, image, rows, cols, ch, out, out_cap, out_cols,
                         out_rows, out_is_obb);
}

// ---- SFSORT (reference ABI) -------------------------------------------------------------------------------
// The python float a float32 configuration member stands for: the shortest decimal that rounds to it (0.6f -> 0.6),
// so thresholds compare as the Python class's do
static double py_float(float f) {
    char buf[32];
    for (int p = 6; p < 10; ++p) {
        snprintf(buf, sizeof(buf), "%.*g", p, (double)f);
        if (strtof(buf, nullptr) == f) return strtod(buf, nullptr);
    }
    return (double)f;
}
BoxMOTSFSORTHandle* boxmot_sfsort_create(const BoxMOTSFSORTConfig* c) {
    Engine* e = nullptr;
    guard([&] {
        if (!c) throw std::runtime_error("NULL config");
        BoxMOTB200TrackerConfig p{};
        p.tracker = BOXMOT_B200_TRACKER_SFSORT;
        p.n_streams = 1;
        p.cap_tracks = 1024;   // the SFSORT class's defaults (boxmot_b200/trackers.py)
        p.cap_dets = 1024;
        p.frame_rate = c->frame_rate;
        p.sf_high_th = py_float(c->high_th);
        p.sf_match_th_first = py_float(c->match_th_first);
        p.sf_new_track_th = py_float(c->new_track_th);
        p.sf_low_th = py_float(c->low_th);
        p.sf_match_th_second = py_float(c->match_th_second);
        p.sf_dynamic_tuning = c->dynamic_tuning;
        p.sf_cth = py_float(c->cth);
        p.sf_high_th_m = py_float(c->high_th_m);
        p.sf_new_track_th_m = py_float(c->new_track_th_m);
        p.sf_match_th_first_m = py_float(c->match_th_first_m);
        p.sf_marginal_timeout = c->marginal_timeout;
        p.sf_central_timeout = c->central_timeout;
        p.sf_frame_width = c->frame_width;
        p.sf_frame_height = c->frame_height;
        p.sf_horizontal_margin = c->horizontal_margin;
        p.sf_vertical_margin = c->vertical_margin;
        e = new Engine(p);
    });
    return reinterpret_cast<BoxMOTSFSORTHandle*>(e);
}
void boxmot_sfsort_destroy(BoxMOTSFSORTHandle* h) { guard([&] { delete reinterpret_cast<Engine*>(h); }); }
int boxmot_sfsort_reset(BoxMOTSFSORTHandle* h) { return guard([&] { as_engine(h)->reset(); }); }
int boxmot_sfsort_update(BoxMOTSFSORTHandle* h, const float* dets, int det_rows, int det_cols, const uint8_t* image,
                         int rows, int cols, int ch, float* out, int out_cap, int out_cols, int* out_rows, int* out_is_obb) {
    return single_update(h, dets, det_rows, det_cols, nullptr, 0, 0, image, rows, cols, ch, out, out_cap, out_cols,
                         out_rows, out_is_obb);
}

// crop staging by name (reid/core/preprocessing.py:47-50).  NULL means "resize_pad" exactly as in the reference's native
// ABI (base/src/reid_capi.cpp:83, botsort/src/c_api.cpp:35); its Python loaders always pass a name (default "resize").
static int preprocess_mode(const char* name) {
    if (!name || !name[0] || strcmp(name, "resize_pad") == 0) return 1;
    if (strcmp(name, "resize") == 0) return 0;
    throw std::runtime_error(std::string("unknown ReID preprocess '") + name + "' (resize, resize_pad)");
}

// ---- BoT-SORT (reference ABI) ------------------------------------------------------------------------------
BoxMOTBotSortHandle* boxmot_botsort_create(const BoxMOTBotSortConfig* c) {
    Engine* e = nullptr;
    guard([&] {
        if (!c) throw std::runtime_error("NULL config");
        if (cmc_requested(c->cmc_method) && strcmp(c->cmc_method, "ecc") != 0)
            throw std::runtime_error("only the 'ecc' camera-motion estimator runs on the device: pass cmc_method=\"ecc\" or NULL "
                                     "(warps of other estimators can be supplied through boxmot_b200_tracker_set_warp)");
        const int prep = preprocess_mode(c->reid_preprocess);
        BoxMOTB200TrackerConfig p{};
        p.tracker = BOXMOT_B200_TRACKER_BOTSORT;
        p.n_streams = 1;
        p.cap_tracks = 2048;
        p.cap_dets = 1024;
        p.feat_dim = 512;
        p.track_buffer = c->track_buffer;
        p.frame_rate = c->frame_rate;
        p.with_reid = c->with_reid;
        p.fuse_first_associate = c->fuse_first_associate;
        p.removed_stracks_buffer = 100;    // botsort.py:85 constructor default
        p.track_high_thresh = c->track_high_thresh;
        p.track_low_thresh = c->track_low_thresh;
        p.new_track_thresh = c->new_track_thresh;
        p.match_thresh = c->match_thresh;
        p.second_match_thresh = 0.5;       // botsort.py:82-84 constructor defaults
        p.unconfirmed_match_thresh = 0.7;
        p.unconfirmed_emb_scale = 2.0;
        p.proximity_thresh = c->proximity_thresh;
        p.appearance_thresh = c->appearance_thresh;
        p.reid_model_path = c->reid_model_path;
        p.reid_preprocess = prep;
        e = new Engine(p);
        if (cmc_requested(c->cmc_method)) {
            try { e->set_cmc(c->cmc_method); } catch (...) { delete e; e = nullptr; throw; }
        }
    });
    return reinterpret_cast<BoxMOTBotSortHandle*>(e);
}
void boxmot_botsort_destroy(BoxMOTBotSortHandle* h) { guard([&] { delete reinterpret_cast<Engine*>(h); }); }
int boxmot_botsort_reset(BoxMOTBotSortHandle* h) { return guard([&] { as_engine(h)->reset(); }); }
int boxmot_botsort_update(BoxMOTBotSortHandle* h, const float* dets, int det_rows, int det_cols, const float* embs,
                          int emb_rows, int emb_cols, const uint8_t* image, int rows, int cols, int ch, float* out,
                          int out_cap, int out_cols, int* out_rows, int* out_is_obb) {
    return single_update(h, dets, det_rows, det_cols, embs, emb_rows, emb_cols, image, rows, cols, ch, out, out_cap,
                         out_cols, out_rows, out_is_obb);
}
int boxmot_botsort_last_reid_time_ms(BoxMOTBotSortHandle* h, double* out) {
    return guard([&] { *out = as_engine(h)->last_reid_ms; });
}
int boxmot_botsort_last_reid_preprocess_time_ms(BoxMOTBotSortHandle* h, double* out) {
    return guard([&] { (void)as_engine(h); *out = 0.0; });  // crop staging is fused into the ReID launch sequence
}
int boxmot_botsort_last_reid_process_time_ms(BoxMOTBotSortHandle* h, double* out) {
    return guard([&] { *out = as_engine(h)->last_reid_ms; });
}
int boxmot_botsort_last_reid_postprocess_time_ms(BoxMOTBotSortHandle* h, double* out) {
    return guard([&] { (void)as_engine(h); *out = 0.0; });
}

// ---- standalone kernels ----------------------------------------------------------------------------------------
int boxmot_b200_jv_dense(const double* cost, int rows, int cols, int* x, int* y) {
    return guard([&] { standalone_jv(cost, rows, cols, x, y); });
}
int boxmot_b200_cmc_ecc(const uint8_t* prev_bgr, const uint8_t* cur_bgr, int rows, int cols, double scale, double eps,
                        int max_iter, float* warp2x3, int* status, uint8_t* prepared) {
    return guard([&] {
        if (!prev_bgr || !cur_bgr || !warp2x3) throw std::runtime_error("NULL argument");
        standalone_ecc(prev_bgr, cur_bgr, rows, cols, scale, eps, max_iter, warp2x3, status, prepared);
    });
}
BoxMOTB200CmcSof* boxmot_b200_cmc_sof_create(double scale, int min_inliers, double min_inlier_ratio,
                                             double ransac_reproj_threshold) {
    void* h = nullptr;
    guard([&] { h = sof_create(scale, min_inliers, min_inlier_ratio, ransac_reproj_threshold); });
    return reinterpret_cast<BoxMOTB200CmcSof*>(h);
}
int boxmot_b200_cmc_sof_apply(BoxMOTB200CmcSof* handle, const uint8_t* bgr, int rows, int cols, const float* dets_xyxy,
                              int n_dets, float* warp2x3, int* status) {
    return guard([&] {
        if (!handle || !bgr || !warp2x3) throw std::runtime_error("NULL argument");
        sof_apply(handle, bgr, rows, cols, dets_xyxy, n_dets, warp2x3, status);
    });
}
void boxmot_b200_cmc_sof_destroy(BoxMOTB200CmcSof* handle) {
    guard([&] { sof_destroy(handle); });
}
int boxmot_b200_jv_dense_mode(int cta_wide) {
    return guard([&] { set_jv_wide(cta_wide); });
}
int boxmot_b200_lsa_solve(const double* cost, int rows, int cols, int* row_ind, int* col_ind, int* out_pairs) {
    return guard([&] {
        const int n = standalone_lsa(cost, rows, cols, row_ind, col_ind);
        if (out_pairs) *out_pairs = n;
    });
}
int boxmot_b200_lap_solve(const double* cost, int rows, int cols, double cost_limit, int* x, int* y) {
    return guard([&] { standalone_lap(cost, rows, cols, cost_limit, x, y); });
}
int boxmot_b200_kalman_predict(int kind, double* mean, double* cov, const int* tracked, int n) {
    return guard([&] { standalone_kf(0, kind, mean, cov, tracked, nullptr, n); });
}
int boxmot_b200_kalman_update(int kind, double* mean, double* cov, const float* meas, int n) {
    return guard([&] { standalone_kf(1, kind, mean, cov, nullptr, meas, n); });
}
int boxmot_b200_kalman_initiate(int kind, const float* meas, double* mean, double* cov, int n) {
    return guard([&] { standalone_kf(2, kind, mean, cov, nullptr, meas, n); });
}
int boxmot_b200_iou_cost(const double* t, int rows, const float* d, int cols, double* out) {
    return guard([&] { standalone_iou(t, rows, d, cols, out); });
}
int boxmot_b200_pointwise_gemm(const float* a, int m, int k, const float* w, int n, const float* bias,
                               const float* residual, int relu, int use_tensor_cores, float* out, float* elapsed_ms) {
    return guard([&] { standalone_pointwise(a, m, k, w, n, bias, residual, relu, use_tensor_cores, out, elapsed_ms); });
}
int boxmot_b200_instance_norm(const float* x, int n, int h, int w, int c, const float* gamma, const float* beta,
                              const float* residual, int relu, int pool, float* out) {
    return guard([&] { standalone_instance_norm(x, n, h, w, c, gamma, beta, residual, relu, pool, out); });
}
int boxmot_b200_resnet_conv(const float* in0, int n, int h0, int w0, int c0, int k, int stride, const float* in1, int h1,
                            int w1, int c1, int stride1, const float* w, int out_c, const float* bias,
                            const float* residual, int relu, float* out, float* elapsed_ms) {
    return guard([&] {
        standalone_resnet_conv(in0, n, h0, w0, c0, k, stride, in1, h1, w1, c1, stride1, w, out_c, bias, residual, relu,
                               out, elapsed_ms);
    });
}
int boxmot_b200_vit_layernorm(const float* x, int rows, const float* gamma, const float* beta, float* out) {
    return guard([&] { standalone_vit_layernorm(x, rows, gamma, beta, out); });
}
int boxmot_b200_vit_attention(const float* qkv, int n, int tokens, float* out) {
    return guard([&] { standalone_vit_attention(qkv, n, tokens, out, 768); });
}
int boxmot_b200_vit_attention_width(const float* qkv, int n, int tokens, int width, float* out) {
    return guard([&] { standalone_vit_attention(qkv, n, tokens, out, width); });
}
int boxmot_b200_vits_layernorm(const float* x, int rows, const float* gamma, const float* beta, float* out) {
    return guard([&] { standalone_vits_layernorm(x, rows, gamma, beta, out); });
}
int boxmot_b200_vits_ain(const float* x, int n, int tokens, const float* a, const float* b, const float* s, float* out) {
    return guard([&] { standalone_vits_ain(x, n, tokens, a, b, s, out); });
}
int boxmot_b200_vits_head(const float* x, int n, int gh, int gw, int pool, int proj, const float* hw, int n_hw,
                          int normalise, float* out) {
    return guard([&] { standalone_vits_head(x, n, gh, gw, pool, proj, hw, n_hw, normalise, out); });
}
int boxmot_b200_mlfn_group_conv(const float* in, int n, int h, int w, int c, int gw, int stride, const float* weight,
                                const float* bias, const float* gates, float* out) {
    return guard([&] { standalone_mlfn_group_conv(in, n, h, w, c, gw, stride, weight, bias, gates, out); });
}
int boxmot_b200_mlfn_fsm(const float* x, int n, int h, int w, int c, const float* w1, const float* b1, int f0,
                         const float* w2, const float* b2, int f1, const float* w3, const float* b3, float* out) {
    return guard([&] { standalone_mlfn_fsm(x, n, h, w, c, w1, b1, f0, w2, b2, f1, w3, b3, out); });
}
int boxmot_b200_f32_pointwise(const float* a, const float* branches, const float* gates, int n, int hw, int k, int mid,
                              const float* w, int nout, const float* bias, const float* residual, int relu, int off,
                              int count, float* out, int out_floats, int* instance) {
    return guard([&] {
        standalone_f32_pointwise(a, branches, gates, n, hw, k, mid, w, nout, bias, residual, relu, off, count, out, out_floats, instance);
    });
}
int boxmot_b200_f32_lightconv(const float* in, int nb, int n, int h, int w, int c, const float* wpw, const float* wdw,
                              const float* bias, int off, int count, float* out, int out_stride, float* sums,
                              int sums_stride, int* instance) {
    return guard([&] {
        standalone_f32_lightconv(in, nb, n, h, w, c, wpw, wdw, bias, off, count, out, out_stride, sums, sums_stride, instance);
    });
}
int boxmot_b200_f32_lightchain(const float* in, int n, int h, int w, int c, const float* wpw, const float* wdw,
                               const float* bias, int off, int count, float* out, int out_stride, float* sums,
                               int sums_stride, int* instance) {
    return guard([&] {
        standalone_f32_lightchain(in, n, h, w, c, wpw, wdw, bias, off, count, out, out_stride, sums, sums_stride, instance);
    });
}
int boxmot_b200_f32_gates(const float* sums, int n, int tiles, int c, int hid, int hw, const float* w1, const float* b1,
                          const float* w2, const float* b2, int off, int count, float* gates, int gates_floats) {
    return guard([&] {
        standalone_f32_gates(sums, n, tiles, c, hid, hw, w1, b1, w2, b2, off, count, gates, gates_floats);
    });
}
int boxmot_b200_f32_head(const float* x, int n, int hw, int c, const float* wfc, const float* bfc, int feat,
                         const int* rows, int off, int count, float* out, int out_floats, int out_ld) {
    return guard([&] { standalone_f32_head(x, n, hw, c, wfc, bfc, feat, rows, off, count, out, out_floats, out_ld); });
}
int boxmot_b200_f32_map(int op, const float* in, int n, int h, int w, int c, int stride, const float* weight,
                        const float* bias, int off, int count, float* out, int out_floats) {
    return guard([&] { standalone_f32_map(op, in, n, h, w, c, stride, weight, bias, off, count, out, out_floats); });
}
int boxmot_b200_f32_lmbn_head(const float* x, int n, int h, int w, const float* neck, const int* rows, int off,
                              int count, float* pooled, int pooled_floats, float* out, int out_floats, int out_ld) {
    return guard([&] {
        standalone_f32_lmbn_head(x, n, h, w, neck, rows, off, count, pooled, pooled_floats, out, out_floats, out_ld);
    });
}
int boxmot_b200_hacnn_conv(const float* in, int n, int off, int count, int h, int w, int c0, int k, int stride,
                           const float* weight, int N, const float* bias, float* out, int out_ld, int out_off) {
    return guard([&] { standalone_hacnn_conv(in, n, off, count, h, w, c0, k, stride, weight, N, bias, out, out_ld, out_off); });
}
int boxmot_b200_hacnn_map(int op, const float* in, int n, int off, int count, int h, int w, int c, const float* weight,
                          const float* bias, float* out) {
    return guard([&] { standalone_hacnn_map(op, in, n, off, count, h, w, c, weight, bias, out); });
}
int boxmot_b200_hacnn_attention(const float* x, int n, int off, int count, int h, int w, int c, int level,
                                const float* params, float* out, float* s, float* v, float* theta) {
    return guard([&] { standalone_hacnn_attention(x, n, off, count, h, w, c, level, params, out, s, v, theta); });
}
int boxmot_b200_hacnn_stn(const float* src, int n, int off, int count, int H, int W, int C, const float* theta,
                          int level, const float* prev, int lh, int lw, float* out) {
    return guard([&] { standalone_hacnn_stn(src, n, off, count, H, W, C, theta, level, prev, lh, lw, out); });
}
int boxmot_b200_hacnn_head(const float* x3, int n, int off, int count, int hw3, const float* loc, int hwl,
                           const float* wg, const float* bg, const float* wl, const float* bl, const int* rows,
                           int out_rows, float* out, float* v) {
    return guard([&] { standalone_hacnn_head(x3, n, off, count, hw3, loc, hwl, wg, bg, wl, bl, rows, out_rows, out, v); });
}
int boxmot_b200_cosine_cost(const float* a, int rows, const float* b, int cols, int dim, double* out) {
    return guard([&] { standalone_cosine(a, rows, b, cols, dim, out); });
}
}

// ---- ReID (reference ABI: base/include/boxmot/trackers/base/reid_capi.h:36-94) ---------------------------------
namespace {
struct ReidHandle {
    ReidModel* model = nullptr;
    cudaStream_t stream = nullptr;
    uint8_t* d_image = nullptr;
    size_t image_cap = 0;
    CropDesc* d_crops = nullptr;
    int* d_ncrops = nullptr;
    float* d_out = nullptr;
    int cap = 0;
    int staged_n = -1;      // boxes staged by preprocess(); -1 = nothing staged
    int staged_rows = 0, staged_cols = 0;
    bool processed = false;
    std::vector<CropDesc> h_crops;
    std::vector<float> h_out;

    ~ReidHandle() {
        if (stream) cudaStreamSynchronize(stream);
        if (model) reid_free(model);
        cudaFree(d_image); cudaFree(d_crops); cudaFree(d_ncrops); cudaFree(d_out);
        if (stream) cudaStreamDestroy(stream);
    }
};

#define CAPI_CUDA_OK(expr)                                                                  \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) throw std::runtime_error(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

ReidHandle* as_reid(void* h) {
    if (!h) throw std::runtime_error("NULL handle");
    return reinterpret_cast<ReidHandle*>(h);
}

void reid_stage(ReidHandle* r, const float* boxes, int n, const uint8_t* image, int rows, int cols, int ch) {
    if (n < 0) throw std::runtime_error("n_boxes < 0");
    if (n > 0 && !boxes) throw std::runtime_error("boxes_xyxy is NULL");
    if (!image || rows <= 0 || cols <= 0) throw std::runtime_error("image is NULL or empty");
    if (ch != 3) throw std::runtime_error("image_channels must be 3 (HxWx3 uint8 BGR)");
    const size_t ib = (size_t)rows * cols * 3;
    if (ib > r->image_cap) {
        cudaFree(r->d_image); r->d_image = nullptr;
        CAPI_CUDA_OK(cudaMalloc(&r->d_image, ib));
        r->image_cap = ib;
    }
    if (n > r->cap) {
        cudaFree(r->d_crops); cudaFree(r->d_out); r->d_crops = nullptr; r->d_out = nullptr;
        int cap = n < 64 ? 64 : n;
        CAPI_CUDA_OK(cudaMalloc(&r->d_crops, sizeof(CropDesc) * cap));
        CAPI_CUDA_OK(cudaMalloc(&r->d_out, sizeof(float) * (size_t)cap * reid_feature_dim(r->model)));
        r->cap = cap;
    }
    if (!r->d_ncrops) CAPI_CUDA_OK(cudaMalloc(&r->d_ncrops, sizeof(int)));
    r->h_crops.resize(n);
    for (int i = 0; i < n; ++i) {
        CropDesc c;
        c.x1 = boxes[i * 4 + 0]; c.y1 = boxes[i * 4 + 1]; c.x2 = boxes[i * 4 + 2]; c.y2 = boxes[i * 4 + 3];
        c.image = 0; c.out_row = i;
        r->h_crops[i] = c;
    }
    CAPI_CUDA_OK(cudaMemcpyAsync(r->d_image, image, ib, cudaMemcpyHostToDevice, r->stream));
    if (n) CAPI_CUDA_OK(cudaMemcpyAsync(r->d_crops, r->h_crops.data(), sizeof(CropDesc) * n, cudaMemcpyHostToDevice, r->stream));
    CAPI_CUDA_OK(cudaMemcpyAsync(r->d_ncrops, &n, sizeof(int), cudaMemcpyHostToDevice, r->stream));
    CAPI_CUDA_OK(cudaStreamSynchronize(r->stream));  // host buffers are borrowed for the call only
    r->staged_n = n; r->staged_rows = rows; r->staged_cols = cols; r->processed = false;
}

void reid_run(ReidHandle* r) {
    if (r->staged_n < 0) throw std::runtime_error("process() called before preprocess()");
    if (r->staged_n > 0)
        reid_forward(r->model, r->d_image, r->image_cap, r->staged_rows, r->staged_cols, r->d_crops, r->d_ncrops,
                     r->staged_n, r->d_out, reid_feature_dim(r->model), r->stream);
    CAPI_CUDA_OK(cudaStreamSynchronize(r->stream));
    r->processed = true;
}

void reid_collect(ReidHandle* r, float* out, int cap_floats) {
    if (!r->processed) throw std::runtime_error("postprocess() called before process()");
    const size_t need = (size_t)r->staged_n * reid_feature_dim(r->model);
    if ((size_t)cap_floats < need) throw std::runtime_error("out_capacity_floats too small");
    if (need) {
        if (!out) throw std::runtime_error("out_features is NULL");
        CAPI_CUDA_OK(cudaMemcpy(out, r->d_out, sizeof(float) * need, cudaMemcpyDeviceToHost));
    }
    r->staged_n = -1; r->processed = false;
}
}  // namespace

extern "C" {
const char* boxmot_reid_capi_last_error(void) { return g_error.c_str(); }

int boxmot_reid_capi_create(const char* model_path, const char* preprocess, void** out_handle) {
    return guard([&] {
        if (!out_handle) throw std::runtime_error("out_handle is NULL");
        *out_handle = nullptr;
        if (!model_path) throw std::runtime_error("model_path is NULL");
        const int prep = preprocess_mode(preprocess);
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
            throw std::runtime_error("no CUDA device: boxmot_b200 has no CPU fallback");
        ReidHandle* r = new ReidHandle();
        try {
            r->model = reid_load(model_path);
            reid_set_preprocess(r->model, prep);
            CAPI_CUDA_OK(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
        } catch (...) {
            delete r;
            throw;
        }
        *out_handle = r;
    });
}
void boxmot_reid_capi_destroy(void* h) { guard([&] { delete reinterpret_cast<ReidHandle*>(h); }); }
int boxmot_reid_capi_feature_dim(void* h, int* out_dim) {
    return guard([&] {
        if (!out_dim) throw std::runtime_error("out_feature_dim is NULL");
        *out_dim = reid_feature_dim(as_reid(h)->model);
    });
}
int boxmot_reid_capi_compute_features(void* h, const float* boxes, int n, const uint8_t* image, int rows, int cols,
                                      int ch, float* out, int cap_floats) {
    return guard([&] {
        ReidHandle* r = as_reid(h);
        reid_stage(r, boxes, n, image, rows, cols, ch);
        reid_run(r);
        reid_collect(r, out, cap_floats);
    });
}
int boxmot_reid_capi_preprocess(void* h, const float* boxes, int n, const uint8_t* image, int rows, int cols, int ch) {
    return guard([&] { reid_stage(as_reid(h), boxes, n, image, rows, cols, ch); });
}
int boxmot_reid_capi_process(void* h) { return guard([&] { reid_run(as_reid(h)); }); }
int boxmot_b200_reid_debug_stage(void* h, const float* boxes, int n, const uint8_t* image, int rows, int cols,
                                 int stage, float* out, int cap_floats, int* floats_per_crop) {
    return guard([&] {
        ReidHandle* r = as_reid(h);
        reid_stage(r, boxes, n, image, rows, cols, 3);
        reid_set_debug_stop(r->model, stage);
        try { reid_run(r); } catch (...) { reid_set_debug_stop(r->model, -1); throw; }
        reid_set_debug_stop(r->model, -1);
        size_t per = 0;
        const float* t = reid_debug_tensor(r->model, &per);
        if (!t) throw std::runtime_error("stage index out of range");
        if (floats_per_crop) *floats_per_crop = (int)per;
        if ((size_t)cap_floats < per * (size_t)n) throw std::runtime_error("out capacity too small");
        CAPI_CUDA_OK(cudaMemcpy(out, t, sizeof(float) * per * n, cudaMemcpyDeviceToHost));
        r->staged_n = -1; r->processed = false;
    });
}
int boxmot_reid_capi_postprocess(void* h, float* out, int cap_floats) {
    return guard([&] { reid_collect(as_reid(h), out, cap_floats); });
}
}
