/*
 * boxmot_b200.h -- C ABI of libboxmot_b200.so: the H100-native drop-in for BoxMOT's per-frame track-update
 * hot path (ReID embedding CNN over detection crops, batched Kalman predict/update, IoU + cosine cost build and
 * linear assignment), sm_90a CUDA behind plain-C entry points (pointers and sizes only; no torch types).
 *
 * Part 1 re-exports, symbol for symbol, the C ABI the reference's ctypes loaders bind
 * (paths relative to /root/reference/boxmot/native/cpp/trackers):
 *   - base/include/boxmot/trackers/base/reid_capi.h:36-94      boxmot_reid_capi_*
 *   - bytetrack/include/bytetrack/c_api.hpp:17-46              boxmot_bytetrack_*
 *   - botsort/include/botsort/c_api.hpp:17-61                  boxmot_botsort_*
 * Same argument meaning, same return convention (int 1 = ok / 0 = failure, NULL handle on failed create,
 * message via the thread-local *_last_error()), caller owns every buffer, 9-column output rows.
 * Semantics follow the reference PYTHON trackers (the oracle of record, SURVEY.md notes N1-N3), not the
 * reference's C++ re-implementation.
 *
 * Part 2 is the append-only B200 extension: double-precision thresholds and the Python-only parameters the
 * reference ABI cannot carry, multi-stream batched updates (one launch per frame for all streams resident
 * on the GPU), device-resident inputs, and standalone entry points for the Kalman / cost / assignment
 * kernels used by the parity tests and the benchmark.
 */
#ifndef BOXMOT_B200_H_
#define BOXMOT_B200_H_

#include <stdint.h>

#if defined(__cplusplus)
extern "C" {
#endif

#define BOXMOT_B200_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------ */
/* Part 1a: ReID (replaces base/include/boxmot/trackers/base/reid_capi.h:36-94)                     */
/* model_path: a `.b200reid` weight blob written by boxmot_b200.weights.export_blob (BN folded), the  */
/* analogue of the reference's .pt -> .onnx auto-export (native/_common.py:453-570).                  */
/* ------------------------------------------------------------------------------------------------ */
BOXMOT_B200_API int boxmot_reid_capi_create(const char* model_path, const char* preprocess, void** out_handle);
BOXMOT_B200_API void boxmot_reid_capi_destroy(void* handle);
BOXMOT_B200_API int boxmot_reid_capi_feature_dim(void* handle, int* out_feature_dim);
BOXMOT_B200_API int boxmot_reid_capi_compute_features(void* handle, const float* boxes_xyxy, int n_boxes,
                                                      const uint8_t* image_data, int image_rows, int image_cols,
                                                      int image_channels, float* out_features,
                                                      int out_capacity_floats);
BOXMOT_B200_API int boxmot_reid_capi_preprocess(void* handle, const float* boxes_xyxy, int n_boxes,
                                                const uint8_t* image_data, int image_rows, int image_cols,
                                                int image_channels);
BOXMOT_B200_API int boxmot_reid_capi_process(void* handle);
BOXMOT_B200_API int boxmot_reid_capi_postprocess(void* handle, float* out_features, int out_capacity_floats);
BOXMOT_B200_API const char* boxmot_reid_capi_last_error(void);

/* ------------------------------------------------------------------------------------------------ */
/* Part 1b: ByteTrack (replaces bytetrack/include/bytetrack/c_api.hpp:17-46)                         */
/* ------------------------------------------------------------------------------------------------ */
typedef struct BoxMOTByteTrackConfig {
    float min_conf;
    float track_thresh;
    float match_thresh;
    int track_buffer;
    int frame_rate;
    int max_obs;
} BoxMOTByteTrackConfig;

typedef struct BoxMOTByteTrackHandle BoxMOTByteTrackHandle;

BOXMOT_B200_API BoxMOTByteTrackHandle* boxmot_bytetrack_create(const BoxMOTByteTrackConfig* config);
BOXMOT_B200_API void boxmot_bytetrack_destroy(BoxMOTByteTrackHandle* handle);
BOXMOT_B200_API int boxmot_bytetrack_reset(BoxMOTByteTrackHandle* handle);
BOXMOT_B200_API int boxmot_bytetrack_update(BoxMOTByteTrackHandle* handle, const float* dets, int det_rows,
                                            int det_cols, const uint8_t* image_data, int image_rows,
                                            int image_cols, int image_channels, float* out_tracks,
                                            int out_capacity_rows, int out_cols, int* out_rows, int* out_is_obb);
BOXMOT_B200_API const char* boxmot_bytetrack_last_error(void);

/* ------------------------------------------------------------------------------------------------ */
/* Part 1c: BoT-SORT (replaces botsort/include/botsort/c_api.hpp:17-61)                              */
/* ------------------------------------------------------------------------------------------------ */
typedef struct BoxMOTBotSortConfig {
    float track_high_thresh;
    float track_low_thresh;
    float new_track_thresh;
    int track_buffer;
    float match_thresh;
    float proximity_thresh;
    float appearance_thresh;
    const char* cmc_method; /* "ecc" runs on the device; NULL, "" or "none" = off (sof / orb / sift: supply the warp) */
    int frame_rate;
    int fuse_first_associate;
    int with_reid;
    int max_obs;
    const char* reid_model_path; /* .b200reid blob, or NULL when embeddings are always passed in */
    const char* reid_preprocess; /* "resize", "resize_pad"; NULL = "resize_pad" as in botsort/src/c_api.cpp:35 */
} BoxMOTBotSortConfig;

typedef struct BoxMOTBotSortHandle BoxMOTBotSortHandle;

BOXMOT_B200_API BoxMOTBotSortHandle* boxmot_botsort_create(const BoxMOTBotSortConfig* config);
BOXMOT_B200_API void boxmot_botsort_destroy(BoxMOTBotSortHandle* handle);
BOXMOT_B200_API int boxmot_botsort_reset(BoxMOTBotSortHandle* handle);
BOXMOT_B200_API int boxmot_botsort_update(BoxMOTBotSortHandle* handle, const float* dets, int det_rows,
                                          int det_cols, const float* embs, int emb_rows, int emb_cols,
                                          const uint8_t* image_data, int image_rows, int image_cols,
                                          int image_channels, float* out_tracks, int out_capacity_rows,
                                          int out_cols, int* out_rows, int* out_is_obb);
BOXMOT_B200_API int boxmot_botsort_last_reid_time_ms(BoxMOTBotSortHandle* handle, double* out_reid_time_ms);
BOXMOT_B200_API int boxmot_botsort_last_reid_preprocess_time_ms(BoxMOTBotSortHandle* handle, double* out_time_ms);
BOXMOT_B200_API int boxmot_botsort_last_reid_process_time_ms(BoxMOTBotSortHandle* handle, double* out_time_ms);
BOXMOT_B200_API int boxmot_botsort_last_reid_postprocess_time_ms(BoxMOTBotSortHandle* handle, double* out_time_ms);
BOXMOT_B200_API const char* boxmot_botsort_last_error(void);

/* SFSORT (sfsort/include/sfsort/c_api.hpp): the configuration member for member.  frame_rate and max_obs are accepted and
 * unused, as there; frame_width / frame_height of 0 take the margins from the first frame's size.  Results follow the
 * Python class (0-based ids); float members stand for the python float they print as (0.6f is 0.6).  det_cols must be
 * 6 (OBB is out of scope); out_is_obb is always 0.  The handle holds 1024 tracks and 1024 detections per frame; lapjv's
 * square problem takes 8 * (1024 + 1024)^2 bytes (34 MB) of device memory. */
typedef struct BoxMOTSFSORTConfig {
    float high_th;
    float match_th_first;
    float new_track_th;
    float low_th;
    float match_th_second;
    int dynamic_tuning;
    float cth;
    float high_th_m;
    float new_track_th_m;
    float match_th_first_m;
    float obb_theta_damping;
    int marginal_timeout;
    int central_timeout;
    int frame_width;
    int frame_height;
    int horizontal_margin;
    int vertical_margin;
    int frame_rate;
    int max_obs;
} BoxMOTSFSORTConfig;

typedef struct BoxMOTSFSORTHandle BoxMOTSFSORTHandle;

BOXMOT_B200_API BoxMOTSFSORTHandle* boxmot_sfsort_create(const BoxMOTSFSORTConfig* config);
BOXMOT_B200_API void boxmot_sfsort_destroy(BoxMOTSFSORTHandle* handle);
BOXMOT_B200_API int boxmot_sfsort_reset(BoxMOTSFSORTHandle* handle);
BOXMOT_B200_API int boxmot_sfsort_update(BoxMOTSFSORTHandle* handle, const float* dets, int det_rows, int det_cols,
                                         const uint8_t* image_data, int image_rows, int image_cols, int image_channels,
                                         float* out_tracks, int out_capacity_rows, int out_cols, int* out_rows,
                                         int* out_is_obb);
BOXMOT_B200_API const char* boxmot_sfsort_last_error(void);

/* ------------------------------------------------------------------------------------------------ */
/* Part 2: B200 extension                                                                            */
/* ------------------------------------------------------------------------------------------------ */
#define BOXMOT_B200_TRACKER_BYTETRACK 0
#define BOXMOT_B200_TRACKER_BOTSORT 1
#define BOXMOT_B200_TRACKER_DEEPOCSORT 2
#define BOXMOT_B200_TRACKER_STRONGSORT 3
#define BOXMOT_B200_TRACKER_BOOSTTRACK 4
#define BOXMOT_B200_TRACKER_OCCLUBOOST 5
#define BOXMOT_B200_TRACKER_SFSORT 6

/* Every parameter of the reference Python constructors (bytetrack.py:226-257, botsort.py:66-118), in
 * double precision so thresholds compare exactly as python floats do. */
typedef struct BoxMOTB200TrackerConfig {
    int tracker;                 /* BOXMOT_B200_TRACKER_* */
    int n_streams;               /* independent streams resident in this handle (>= 1) */
    int cap_tracks;              /* per-stream track slots (active + lost + births of one frame) */
    int cap_dets;                /* per-stream detections per frame */
    int feat_dim;                /* embedding width when with_reid (512 OSNet, 1792 MobileNetV2) */
    int track_buffer;
    int frame_rate;
    int with_reid;
    int fuse_first_associate;
    int removed_stracks_buffer;  /* BoT-SORT deque(maxlen); ignored by ByteTrack (unbounded list) */
    double track_high_thresh;    /* ByteTrack: track_thresh */
    double track_low_thresh;     /* ByteTrack: min_conf */
    double new_track_thresh;     /* ByteTrack: det_thresh == track_thresh */
    double match_thresh;
    double second_match_thresh;       /* ByteTrack: 0.5 */
    double unconfirmed_match_thresh;  /* ByteTrack: 0.7 */
    double proximity_thresh;
    double appearance_thresh;
    double unconfirmed_emb_scale;
    const char* reid_model_path; /* optional .b200reid blob: ReID runs on-device inside update() */
    /* DeepOCSORT (trackers/bbox/deepocsort/deepocsort.py:263-300 + BaseTracker det_thresh / max_age / min_hits /
     * iou_threshold); ignored by the other trackers */
    int delta_t;
    int max_age;
    int min_hits;
    int embedding_off;
    int aw_off;
    double det_thresh;
    double iou_threshold;
    double inertia;
    double w_association_emb;
    double alpha_fixed_emb;
    double aw_param;
    double q_xy_scaling;
    double q_s_scaling;
    /* StrongSORT (trackers/bbox/strongsort/strongsort.py:38-67; max_age above is shared); ignored by the others */
    int n_init;
    int nn_budget;               /* samples kept per track (the reference's None = unbounded is not supported) */
    double min_conf;
    double max_cos_dist;
    double max_iou_dist;
    double mc_lambda;
    double ema_alpha;
    /* crop staging of the on-device ReID (reid/core/preprocessing.py): 0 = "resize" (the Python default), 1 = "resize_pad"
     * (aspect-preserving resize + ImageNet-mean border, the native default when the name is NULL) */
    int reid_preprocess;
    /* BoostTrack / BoostTrack++ (trackers/bbox/boosttrack/boosttrack.py:241-296; det_thresh, max_age, min_hits,
     * iou_threshold and with_reid above are shared); ignored by the other trackers */
    int use_dlo_boost;
    int use_duo_boost;
    int use_rich_s;
    int use_sb;
    int use_vt;
    int s_sim_corr;
    double dlo_boost_coef;
    double lambda_iou;
    double lambda_mhd;
    double lambda_shape;
    double min_box_area;
    double aspect_ratio_thresh;
    /* OccluBoost (trackers/bbox/occluboost/occluboost.py:84-183; the BoostTrack fields above are shared, and so are
     * track_low_thresh and new_track_thresh); ignored by the other trackers.  Values as the reference stores them
     * after its clamps (confirm_hits >= 1, tentative_max_age >= 0, ams_buffer_size >= 2, gta_min_track_length >= 1,
     * gta_max_gap >= 1, ams_alpha0 and ams_shrink_ratio in [0, 1], ams_threshold >= 0, new_track_thresh >= 0). */
    int use_second_pass;
    int recovery_max_age;
    int second_pass_max_age;
    int second_pass_min_hits;
    int confirm_hits;
    int tentative_max_age;
    int ams_enabled;
    int ams_buffer_size;
    int gta_enabled;
    int gta_min_track_length;
    int gta_max_gap;
    double lambda_emb_multiplier;
    double recovery_appearance_thresh;
    double recovery_iou_thresh;
    double feat_alpha;
    double second_iou_thresh;
    double second_appearance_thresh;
    double instant_confirm_thresh;
    double duplicate_iou_thresh;
    double ams_alpha0;
    double ams_threshold;
    double ams_shrink_ratio;
    double gta_appearance_thresh;
    /* SFSORT (sfsort.py:180-237); the engine applies the constructor's clamps.  frame_width / frame_height of 0: the
     * margins come from the first frame's size. */
    double sf_high_th;
    double sf_match_th_first;
    double sf_new_track_th;
    double sf_low_th;
    double sf_match_th_second;
    int sf_dynamic_tuning;
    double sf_cth;
    double sf_high_th_m;
    double sf_new_track_th_m;
    double sf_match_th_first_m;
    int sf_marginal_timeout;
    int sf_central_timeout;
    int sf_frame_width;
    int sf_frame_height;
    double sf_horizontal_margin;
    double sf_vertical_margin;
    /* log10(k) for k = 0 .. sf_log10_count - 1 (at least cap_dets + 1 entries), the value the density-tuned thresholds
     * use for k scores above cth; the Python layer passes numpy's.  NULL: the host libm's log10. */
    const double* sf_log10_table;
    int sf_log10_count;
} BoxMOTB200TrackerConfig;

typedef struct BoxMOTB200Tracker BoxMOTB200Tracker;

BOXMOT_B200_API BoxMOTB200Tracker* boxmot_b200_tracker_create(const BoxMOTB200TrackerConfig* config);
BOXMOT_B200_API void boxmot_b200_tracker_destroy(BoxMOTB200Tracker* handle);
BOXMOT_B200_API int boxmot_b200_tracker_reset(BoxMOTB200Tracker* handle);

/* One frame for every stream of the handle in a single launch sequence.
 *   dets[s]      (det_rows[s], 6) float32 host rows [x1,y1,x2,y2,conf,cls]; may be NULL when det_rows[s]==0
 *   embs[s]      (det_rows[s], feat_dim) float32 host rows, or embs == NULL / embs[s] == NULL
 *   images[s]    H x W x 3 uint8 BGR host frame (only read when ReID runs inside the call)
 *   out[s]       (out_capacity_rows[s], 9) float32; rows [x1,y1,x2,y2,id,conf,cls,det_ind,0]
 * Per-stream results equal `n_streams` independent reference trackers. */
BOXMOT_B200_API int boxmot_b200_tracker_update_batch(BoxMOTB200Tracker* handle, const float* const* dets,
                                                     const int* det_rows, const float* const* embs,
                                                     const uint8_t* const* images, int image_rows,
                                                     int image_cols, float* const* out,
                                                     const int* out_capacity_rows, int* out_rows);

/* Device-resident variant for pipelines that keep frames and detections in HBM (and for the benchmark's
 * kernel-only figure): d_dets is [n_streams][cap_dets][6] float32, d_embs [n_streams][cap_dets][feat_dim] or
 * NULL, d_images [n_streams][rows*cols*3] or NULL, det_rows on the host.  Results are left in device memory
 * ([n_streams][cap_dets][8] rows + counts) and copied out by boxmot_b200_tracker_fetch. `sync` = 0 returns
 * right after enqueueing. */
BOXMOT_B200_API int boxmot_b200_tracker_update_device(BoxMOTB200Tracker* handle, const float* d_dets,
                                                      const int* det_rows, const float* d_embs,
                                                      const uint8_t* d_images, int image_rows, int image_cols,
                                                      int sync);
BOXMOT_B200_API int boxmot_b200_tracker_fetch(BoxMOTB200Tracker* handle, float* const* out,
                                              const int* out_capacity_rows, int* out_rows);

/* Test / diagnostics: live track ids with their Kalman mean (8) and covariance (64), float64. */
BOXMOT_B200_API int boxmot_b200_tracker_snapshot(BoxMOTB200Tracker* handle, int stream, int* ids, double* means,
                                                 double* covs, int capacity, int* out_count);
/* Ids of one of the tracker's lists in list order: which = 0 active, 1 lost, 2 removed -- what the reference exposes as
 * BaseTracker.active_tracks / lost_stracks / removed_stracks (boxmot/trackers/basetracker.py:386-390, 465-466). */
BOXMOT_B200_API int boxmot_b200_tracker_track_ids(BoxMOTB200Tracker* handle, int stream, int which, int* ids,
                                                  int capacity, int* out_count);
/* OccluBoost: the graveyard resurrections of `stream` logged since the last call, oldest first, OB_EV = 13 doubles
 * each: grave id, death frame, resurrection frame, box at death [x1,y1,x2,y2], box of the new track, conf and cls at
 * death -- what trackers/bbox/occluboost/occluboost.py:680-698 interpolates into gap rows.  The log is cleared;
 * clear_graveyard != 0 also empties the graveyard (flush_gta, occluboost.py:727-728).  Synchronises the handle. */
BOXMOT_B200_API int boxmot_b200_tracker_gta_events(BoxMOTB200Tracker* handle, int stream, int clear_graveyard,
                                                   double* events, int capacity, int* out_count);
/* Kernel launches issued by the last update call, and CUDA stream / device-time accessors for benchmarks. */
BOXMOT_B200_API int boxmot_b200_tracker_last_launches(BoxMOTB200Tracker* handle, int* out_launches);
BOXMOT_B200_API int boxmot_b200_tracker_last_device_ms(BoxMOTB200Tracker* handle, double* reid_ms, double* assoc_ms);
/* Camera-motion compensation with a SUPPLIED 2x3 warp (row major, float64), applied once, on the next update:
 * BoT-SORT to the predicted pool and the unconfirmed tracks exactly as STrack.multi_gmc does
 * (trackers/bbox/botsort/botsort_track.py:117-132); StrongSORT through Track.camera_update
 * (trackers/bbox/strongsort/sort/track.py:139-148; without a supplied warp it runs with the identity, as the
 * reference does whenever tracks exist); DeepOCSORT through KalmanBoxTracker.apply_affine_correction before the
 * predict step (trackers/bbox/deepocsort/deepocsort.py:189-206, 345-348; motion/kalman_filters/xysr.py:311-366);
 * BoostTrack through KalmanBoxTracker.camera_update before the predict step (boosttrack.py:132-172, 318-321).
 * A supplied warp is how the estimators that are not built on the device (sof, orb, sift) reach the trackers. */
BOXMOT_B200_API int boxmot_b200_tracker_set_warp(BoxMOTB200Tracker* handle, int stream, const double* warp2x3);
/* Camera-motion ESTIMATION on the device, every frame, from the frame passed to update (SURVEY 8f-3): method "ecc" is
 * the reference's ECC estimator with its defaults -- cv2.findTransformECC translation model, eps 1e-5, 100 iterations,
 * gray registration image at scale 0.15 (boxmot/motion/cmc/ecc.py:23-108, base_cmc.py:29-60) -- as StrongSORT runs it on
 * every frame that starts with tracks (trackers/bbox/strongsort/strongsort.py:67,83-86) and BoT-SORT with
 * cmc_method="ecc" (trackers/bbox/botsort/botsort.py:78,116-117,142) -- BoT-SORT and StrongSORT handles.  Method "sof"
 * is the reference's SOF estimator with its defaults (boxmot/motion/cmc/sof.py; as boxmot_b200_cmc_sof_*) on every
 * frame, with the detection boxes the reference masks: every row for BoT-SORT (botsort.py:301), the rows with
 * conf > det_thresh for DeepOCSORT (deepocsort.py:330-349) -- BoT-SORT and DeepOCSORT handles.  BoostTrack handles
 * take both, run the estimator on every frame with every detection row (boosttrack.py:318-321) and apply its result --
 * the identity when it returns none -- to every track.  "none" / "" / NULL turns it off again.  The estimate replaces a warp supplied for the same frame; reset restarts the estimator. */
BOXMOT_B200_API int boxmot_b200_tracker_set_cmc(BoxMOTB200Tracker* handle, const char* method);
/* SFSORT handles: the size (rows x cols) of one stream's frames.  A stream takes its margins from the first size it is
 * given (the reference's first image); update calls that pass image_rows / image_cols > 0 set every stream's size.
 * Streams of different resolutions in one handle need this call.  Other handles: an error. */
BOXMOT_B200_API int boxmot_b200_tracker_set_frame_size(BoxMOTB200Tracker* handle, int stream, int rows, int cols);
/* Device timing on the handle's own CUDA stream: record mark 0 / mark 1 around a region, then read the elapsed
 * milliseconds (synchronises on mark 1). */
BOXMOT_B200_API int boxmot_b200_tracker_mark(BoxMOTB200Tracker* handle, int which);
BOXMOT_B200_API int boxmot_b200_tracker_elapsed_ms(BoxMOTB200Tracker* handle, double* out_ms);
/* Profiling pass: when enabled every kernel launch is bracketed by CUDA events (frames are serialised).
 * profile_read returns accumulated milliseconds and launch counts for 9 classes:
 * crop, stem, maxpool, pointwise, lightconv, gates, avgpool, head, association (3 kernels) - and resets them. */
/* SM-clock ticks the association kernel spent per phase since the last reset (16 slots; 0 split+predict,
 * 1 cost build, 2 assignment, 3 Kalman update + bookkeeping, 4 second round, 5 unconfirmed round, 6 births +
 * list algebra, 7 duplicate suppression + output). */
BOXMOT_B200_API int boxmot_b200_tracker_phase_clocks(BoxMOTB200Tracker* handle, int stream, long long* out16,
                                                     int reset);
BOXMOT_B200_API int boxmot_b200_tracker_profile(BoxMOTB200Tracker* handle, int enable);
BOXMOT_B200_API int boxmot_b200_tracker_profile_read(BoxMOTB200Tracker* handle, double* ms, int* launches);
BOXMOT_B200_API const char* boxmot_b200_last_error(void);

/* Standalone hot-path kernels (parity tests and micro-benchmarks call these through the same library). */
/* lapjv(extend_cost=True, cost_limit=thresh): cost (T,D) float64 host -> x (T), y (D) int32. */
BOXMOT_B200_API int boxmot_b200_lap_solve(const double* cost, int rows, int cols, double cost_limit, int* x, int* y);
/* lapjv(cost, extend_cost=True) (no cost limit, zero-padded to square) with lapjv's own tie-breaking -- the dense
 * Jonker-Volgenant solver DeepOCSORT's association needs for bit-exact ids. cost (rows, cols) float64 host. */
BOXMOT_B200_API int boxmot_b200_jv_dense(const double* cost, int rows, int cols, int* x, int* y);
/* ECC().apply(prev) followed by ECC().apply(cur) on two BGR frames (rows x cols x 3 uint8, host): the float32 2x3 warp
 * the second call returns (row major), status 0 = estimated, 1 = OpenCV would have raised StsNoConv (identity, as
 * ecc.py:69-79 returns); `prepared` (optional, rint(rows*scale) x rint(cols*scale) uint8) receives the registration
 * image of `cur` (BaseCMC.preprocess). */
BOXMOT_B200_API int boxmot_b200_cmc_ecc(const uint8_t* prev_bgr, const uint8_t* cur_bgr, int rows, int cols, double scale,
                                        double eps, int max_iter, float* warp2x3, int* status, uint8_t* prepared);
/* Standalone SOF estimator: the reference's SOF(scale, min_inliers, min_inlier_ratio, ransac_reproj_threshold) camera-
 * motion estimator (boxmot/motion/cmc/sof.py: corners, cornerSubPix on the initialising frame, pyramidal LK, RANSAC
 * partial affine) running on the device.  One handle is one video: it keeps the previous pyramid and keypoints.
 * apply() takes a BGR frame (rows x cols x 3 uint8, host) and the frame's detection boxes (n_dets x 4 float32 xyxy in
 * frame pixels, host; NULL when n_dets is 0, cleared from the corner mask) and writes the float32 2x3 warp SOF.apply
 * returns (row major).  status: 0 = initialising frame (identity), 1 = estimated, 2 = rejected (identity: too few
 * tracks or inliers).  A new frame size starts the estimator afresh. */
typedef struct BoxMOTB200CmcSof BoxMOTB200CmcSof;
BOXMOT_B200_API BoxMOTB200CmcSof* boxmot_b200_cmc_sof_create(double scale, int min_inliers, double min_inlier_ratio,
                                                             double ransac_reproj_threshold);
BOXMOT_B200_API int boxmot_b200_cmc_sof_apply(BoxMOTB200CmcSof* handle, const uint8_t* bgr, int rows, int cols,
                                              const float* dets_xyxy, int n_dets, float* warp2x3, int* status);
BOXMOT_B200_API void boxmot_b200_cmc_sof_destroy(BoxMOTB200CmcSof* handle);
/* Augmentation variant of the dense solver for this process: 3 = column-owned CTA-wide search with the exact shortcuts
 * (no-op band columns, parallel _find_dense tail, hit list, CTA-wide row reduction; the default), 2 = column-owned
 * (distances in registers), 1 = CTA-wide search over list positions, 0 = one-warp search; values >= 4 are
 * `3 | shortcut bits << 2` for bisecting.  All reproduce lapjv's results, the parity tests run every variant (env
 * BOXMOT_B200_JV_WIDE sets the initial value). */
BOXMOT_B200_API int boxmot_b200_jv_dense_mode(int cta_wide);
/* scipy.optimize.linear_sum_assignment(cost) with scipy's own tie-breaking (StrongSORT's min_cost_matching,
 * trackers/bbox/strongsort/sort/linear_assignment.py:62): cost (rows, cols) float64 host -> min(rows, cols) pairs
 * (row_ind ascending, col_ind), count through out_pairs. */
BOXMOT_B200_API int boxmot_b200_lsa_solve(const double* cost, int rows, int cols, int* row_ind, int* col_ind,
                                          int* out_pairs);
/* batched Kalman steps on host arrays: kind 0 = XYAH, 1 = XYWH; mean (n,8), cov (n,8,8) float64 in place. */
BOXMOT_B200_API int boxmot_b200_kalman_predict(int kind, double* mean, double* cov, const int* tracked, int n);
BOXMOT_B200_API int boxmot_b200_kalman_update(int kind, double* mean, double* cov, const float* meas, int n);
BOXMOT_B200_API int boxmot_b200_kalman_initiate(int kind, const float* meas, double* mean, double* cov, int n);
/* 1 - IoU of float64 track boxes (T,4) against float32 detection boxes (D,4) -> (T,D) float64. */
BOXMOT_B200_API int boxmot_b200_iou_cost(const double* track_xyxy, int rows, const float* det_xyxy, int cols,
                                         double* out);
/* max(0, cosine distance) of float32 rows a (T,F) x b (D,F) -> (T,D) float64. */
BOXMOT_B200_API int boxmot_b200_cosine_cost(const float* a, int rows, const float* b, int cols, int dim, double* out);
/* 1x1 convolution as a GEMM on host arrays: out (M,N) = act(A (M,K) * W (K,N) + bias (+ residual)); K, N multiples
 * of 4.  use_tensor_cores = 1 runs the wgmma tf32x3 kernel (M % 128 == 0), 0 the CUDA-core kernel.  elapsed_ms
 * (optional) receives the average device time of 10 back-to-back launches. */
BOXMOT_B200_API int boxmot_b200_pointwise_gemm(const float* a, int m, int k, const float* w, int n, const float* bias,
                                               const float* residual, int relu, int use_tensor_cores, float* out,
                                               float* elapsed_ms);
/* Instance norm (InstanceNorm2d, affine, eps 1e-5, statistics per crop and channel) of OSNet-AIN / OSNet-IBN on host
 * arrays, x (n,H,W,C) NHWC float32, C a multiple of 4.  pool = 0: out (n,H,W,C) = act(IN(x) * gamma + beta
 * (+ residual, optional)), act = ReLU when relu = 1.  pool = 1: the stem form, out (n,H/2,W/2,C) = 3x3 stride-2
 * max pool of relu(IN(x) * gamma + beta). */
BOXMOT_B200_API int boxmot_b200_instance_norm(const float* x, int n, int h, int w, int c, const float* gamma,
                                              const float* beta, const float* residual, int relu, int pool, float* out);
/* One convolution of the ResNet50 / ResNet101 path (wgmma tf32x3 implicit GEMM) on host arrays, NHWC float32:
 * out (n,Ho,Wo,out_c) = act(conv(in0) + conv1x1(in1) + bias (+ residual, optional)), act = none when relu = 0, ReLU
 * when relu = 1, QuickGELU x * sigmoid(1.702 x) when relu = 2 (CLIP's MLP; a CLIP linear layer is a 1x1 convolution
 * over h0 = tokens, w0 = 1), exact GELU x * (1 + erf(x / sqrt 2)) / 2 when relu = 4 (the ViT-Nano / ViT-Tiny MLP). relu = 3 gives relu(residual + relu(conv(in0) + conv1x1(in1) + bias)) (MLFN's fm_conv3, whose
 * ReLU precedes the residual add; the residual is then required).  in0 (n,h0,w0,c0) is read by a k x k kernel (k 1 or 3, pad k/2) at `stride`; in1 (n,h1,w1,c1), optional (c1 = 0
 * for none), by a 1x1 kernel at `stride1` over the same output grid (the fused conv3 + downsample of a stage's first
 * Bottleneck).  w is (k*k*c0 + c1, out_c) K-major, k index (kh*k + kw)*c0 + ci then the c1 channels; c0 and c1
 * multiples of 32, out_c a multiple of 64.  elapsed_ms (optional) receives the average device time of 10 launches. */
BOXMOT_B200_API int boxmot_b200_resnet_conv(const float* in0, int n, int h0, int w0, int c0, int k, int stride,
                                            const float* in1, int h1, int w1, int c1, int stride1, const float* w,
                                            int out_c, const float* bias, const float* residual, int relu, float* out,
                                            float* elapsed_ms);
/* LayerNorm of the CLIP ViT-B/16 path on host arrays: out (rows,768) = LN(x) * gamma + beta, eps 1e-5, float32. */
BOXMOT_B200_API int boxmot_b200_vit_layernorm(const float* x, int rows, const float* gamma, const float* beta,
                                              float* out);
/* Multi-head attention of the CLIP ViT-B/16 path on host arrays: qkv (n,tokens,2304) holds q | k | v, head h at
 * columns 64h..64h+63 of each, with q already scaled by 1/8; out (n,tokens,768) = softmax(q k^T) v per head, heads
 * interleaved.  1 <= tokens <= 288. */
BOXMOT_B200_API int boxmot_b200_vit_attention(const float* qkv, int n, int tokens, float* out);
/* The same attention at width 768 (12 heads, 1 <= tokens <= 288) or 192 (the ViT-Nano / ViT-Tiny path: 3 heads,
 * 1 <= tokens <= 320): qkv (n,tokens,3 width), out (n,tokens,width). */
BOXMOT_B200_API int boxmot_b200_vit_attention_width(const float* qkv, int n, int tokens, int width, float* out);
/* LayerNorm of the ViT-Nano / ViT-Tiny path on host arrays: out (rows,192) = LN(x) * gamma + beta, eps 1e-5. */
BOXMOT_B200_API int boxmot_b200_vits_layernorm(const float* x, int rows, const float* gamma, const float* beta,
                                               float* out);
/* AdaptiveINLN of the ViT-Nano AIN blocks on host arrays: x (n,tokens,192) -> out = a * IN(x) + b * LN(x) + s per
 * channel, IN over the tokens of each crop (biased variance), LN over the channels of each token, both eps 1e-5 and
 * without affine (a, b, s fold the gate and both affines).  tokens * 192 floats must fit in 200 KB of shared memory. */
BOXMOT_B200_API int boxmot_b200_vits_ain(const float* x, int n, int tokens, const float* a, const float* b,
                                         const float* s, float* out);
/* Head of the ViT-Nano / ViT-Tiny path on host arrays: x (n,1 + gh*gw,192) is the final norm's output; pool 0 takes
 * the class token, 1 the omni-scale aggregation of the patch mean (proj 0), P = 2 or 3 the class token and P grid-row
 * strips (proj 512); hw (n_hw floats) is the head block of the blob.  out (n,feat) is L2-normalised when `normalise`,
 * else the row before the norm. */
BOXMOT_B200_API int boxmot_b200_vits_head(const float* x, int n, int gh, int gw, int pool, int proj, const float* hw,
                                          int n_hw, int normalise, float* out);
/* Grouped 3x3 convolution of the MLFN path (fm_conv2, 32 groups, pad 1) on host arrays, NHWC float32: in (n,h,w,c)
 * with c = 32 gw, group width gw in {4, 8, 16, 32}, stride 1 or 2, output width a multiple of 4; weight (9,gw,c),
 * element (kh*3 + kw, i, co) weighing input channel (co / gw) gw + i; out (n,Ho,Wo,c) = relu(conv + bias) *
 * gates[n][co / gw] with gates (n,32). */
BOXMOT_B200_API int boxmot_b200_mlfn_group_conv(const float* in, int n, int h, int w, int c, int gw, int stride,
                                                const float* weight, const float* bias, const float* gates, float* out);
/* Factor-selection module of the MLFN path on host arrays: x (n,h,w,c) NHWC float32 -> out (n,32) = sigmoid(relu(
 * relu(mean_hw(x) w1 + b1) w2 + b2) w3 + b3), w1 (c,f0), w2 (f0,f1), w3 (f1,32) K-major; c, f0, f1 multiples of 64. */
BOXMOT_B200_API int boxmot_b200_mlfn_fsm(const float* x, int n, int h, int w, int c, const float* w1, const float* b1,
                                         int f0, const float* w2, const float* b2, int f1, const float* w3,
                                         const float* b3, float* out);
/* The HACNN kernels on their own, over a crop window as for the float32 kernels below (n crops in the arrays, device
 * count `count`, window start `off`; every output array uploaded as given and read back whole), NHWC float32.
 * hacnn_conv: one ConvBlock on the tensor cores (the Inception streams' SLICE store): in (n,h,w,c0), c0 a multiple of
 * 32, k 1 or 3 (pad k/2), stride 1 or 2, weight (k*k*c0, N) K-major with k index (kh*k + kw)*c0 + ci, N a multiple of
 * 32; out (n,Ho,Wo,out_ld) columns out_off .. out_off + N - 1 = relu(conv + bias), Ho = (h - 1) / stride + 1.
 * hacnn_map: op 0 the 3x3 stride-2 stem (in (n,160,64,3), weight (27,32) as above, bias (32) -> (n,80,32,32), ReLU),
 * op 1 the 3x3 stride-1 pad-1 average pool (/ 9), op 2 the 3x3 stride-2 pad-1 max pool (odd sizes: Ho = (h - 1) / 2 + 1).
 * hacnn_attention: x (n,h,w,c), even h, w with h w <= 640, c a multiple of 16 up to 384, params the level's attention
 * arrays in blob order (each padded to 4 floats): out = x * sigmoid(relu(s[p] v[o] + bv[o])) with s (n,h*w) the
 * spatial map and v (n,c) = W c, and theta (n,24) columns 8 level .. 8 level + 7 = tanh(fc(mean_hw(x))).
 * hacnn_stn: src (n,H,W,C), theta (n,24) columns 8 level .., prev (n,4,lh,lw,C) or NULL -> out (n,4,lh,lw,C) = the four
 * regions' affine_grid + grid_sample of src (align_corners=False, zero padding), resized to lh x lw with
 * align_corners=True (+ prev).
 * hacnn_head: x3 (n,hw3,384), loc (n,4,hwl,384) -> v (n,1024) = [relu(mean(x3) wg + bg) | relu(mean(loc) wl + bl)]
 * (wg (384,512), wl (1536,512) K-major) and out row rows[off + i] = v_i with each half L2-normalised, then the row. */
BOXMOT_B200_API int boxmot_b200_hacnn_conv(const float* in, int n, int off, int count, int h, int w, int c0, int k,
                                           int stride, const float* weight, int N, const float* bias, float* out,
                                           int out_ld, int out_off);
BOXMOT_B200_API int boxmot_b200_hacnn_map(int op, const float* in, int n, int off, int count, int h, int w, int c,
                                          const float* weight, const float* bias, float* out);
BOXMOT_B200_API int boxmot_b200_hacnn_attention(const float* x, int n, int off, int count, int h, int w, int c,
                                                int level, const float* params, float* out, float* s, float* v,
                                                float* theta);
BOXMOT_B200_API int boxmot_b200_hacnn_stn(const float* src, int n, int off, int count, int H, int W, int C,
                                          const float* theta, int level, const float* prev, int lh, int lw, float* out);
BOXMOT_B200_API int boxmot_b200_hacnn_head(const float* x3, int n, int off, int count, int hw3, const float* loc,
                                           int hwl, const float* wg, const float* bg, const float* wl, const float* bl,
                                           const int* rows, int out_rows, float* out, float* v);
/* The float32 CUDA-core kernels of the OSNet family, MobileNetV2 and LMBN_n, one family per entry, launched as a loaded
 * model launches them, on host arrays (NHWC float32) over a crop window: the arrays hold n crops, the device crop count
 * is `count` and the window starts at crop `off`, so the kernels process crops 0 .. clamp(count - off, 0, n) - 1 of the
 * arrays (head entries: with output rows rows[off + i], rows holding off + n entries).  Every output array is uploaded
 * as given and read back whole (out_floats / *_stride floats per tensor), so values the kernels must not write come
 * back unchanged.  `instance` (optional, 4 ints) receives the kernel instance that ran.
 *   f32_pointwise: out (n,hw,nout) = act(A W + bias (+ residual)), act 0 none, 1 ReLU, 2 ReLU6; branches (4,n,hw,mid)
 *     and gates (n,4,mid) select the gated prologue A = [sum_b gates[crop][b] * branch_b | a (n,hw,k-mid), null when
 *     k == mid], else A = a (n,hw,k).  instance {BN, threads, gated, 0}.
 *   f32_lightconv: nb <= 4 LightConv3x3 branches of one level (1x1 wpw (C,C) -> depthwise 3x3 wdw (9,C) + bias + ReLU),
 *     in (nb,n,h,w,c); branch b writes out + b out_stride and, with sums, its per-tile channel sums (n,h/R,c) at
 *     sums + b sums_stride (strides multiples of 4).  instance {1 generic / 2 shape-specialised kernel, C, W, R (tile rows)}.
 *   f32_lightchain: the four branches of an OSBlock in whole-branch CTAs, in (n,h,w,c), weights of LightConv
 *     l = b (b + 1) / 2 + level - 1 at wpw (10,c,c), wdw (10,9,c), bias (10,c); outputs and sums as f32_lightconv.
 *     instance {3, C, W, R}.
 *   f32_gates: gates (n,4,c) = sigmoid(relu(mean w1 + b1) w2 + b2), mean = sum over tiles of sums (4,n,tiles,c) / hw,
 *     w1 (c,hid), w2 (hid,c).
 *   f32_head: average pool of x (n,hw,c), fc (c,feat) + bias + ReLU (wfc null: feat == c, no fc), L2 norm, into the
 *     rows of out (out_ld floats per row).
 *   f32_map: op 0 7x7/2 stem + bias + ReLU of (n,h,128,3) crops, h 256 or 384, weight (147,c); 1 the same without
 *     bias and ReLU; 2 3x3/2 max pool; 3 2x2/2 average pool; 4 MobileNetV2's 3x3/2 stem + bias + ReLU6 of (n,256,128,3)
 *     crops, weight (27,c); 5 depthwise 3x3 pad 1 at stride 1 or 2 + bias + ReLU6, weight (9,c).
 *   f32_lmbn_head: LMBN_n's poolings of the bottleneck, partial and channel branch maps x (3,n,h,w,512) into pooled
 *     (n,6,512), the neck (neck = reduction weights (5,512,512), biases (5,512), shared (256,512), its bias (512),
 *     reduction_ch scale / shift (4,512)) and the L2 norm of the 3584-d rows. */
BOXMOT_B200_API int boxmot_b200_f32_pointwise(const float* a, const float* branches, const float* gates, int n, int hw,
                                              int k, int mid, const float* w, int nout, const float* bias,
                                              const float* residual, int relu, int off, int count, float* out,
                                              int out_floats, int* instance);
BOXMOT_B200_API int boxmot_b200_f32_lightconv(const float* in, int nb, int n, int h, int w, int c, const float* wpw,
                                              const float* wdw, const float* bias, int off, int count, float* out,
                                              int out_stride, float* sums, int sums_stride, int* instance);
BOXMOT_B200_API int boxmot_b200_f32_lightchain(const float* in, int n, int h, int w, int c, const float* wpw,
                                               const float* wdw, const float* bias, int off, int count, float* out,
                                               int out_stride, float* sums, int sums_stride, int* instance);
BOXMOT_B200_API int boxmot_b200_f32_gates(const float* sums, int n, int tiles, int c, int hid, int hw, const float* w1,
                                          const float* b1, const float* w2, const float* b2, int off, int count,
                                          float* gates, int gates_floats);
BOXMOT_B200_API int boxmot_b200_f32_head(const float* x, int n, int hw, int c, const float* wfc, const float* bfc,
                                         int feat, const int* rows, int off, int count, float* out, int out_floats,
                                         int out_ld);
BOXMOT_B200_API int boxmot_b200_f32_map(int op, const float* in, int n, int h, int w, int c, int stride,
                                        const float* weight, const float* bias, int off, int count, float* out,
                                        int out_floats);
BOXMOT_B200_API int boxmot_b200_f32_lmbn_head(const float* x, int n, int h, int w, const float* neck, const int* rows,
                                              int off, int count, float* pooled, int pooled_floats, float* out,
                                              int out_floats, int out_ld);
BOXMOT_B200_API int boxmot_b200_device_count(void);
/* Diagnostics for the ReID kernels: run the forward up to `stage` (0 input blob, 1 stem, 2 max-pool, 3..10 the
 * six OSBlocks and two transitions in order, 11 conv5) and copy that NHWC float32 tensor of the n crops out.  For
 * OSNet-AIN / OSNet-IBN the stem tap is the map after the instance norm and the ReLU.  For ResNet50 / ResNet101: 0 input
 * blob, 1 stem, 2 max-pool, 3 + i the output of Bottleneck i (layer1.0 first).  For CLIP ViT-B/16: 0 input blob
 * (256 x 128 or 256 x 256), 1 patch embedding (patches x 768), 2 ln_pre (tokens x 768), 3 + l the output of residual
 * block l, 15 the head row before the L2 normalisation (1280).  For MLFN: 0 input blob, 1 stem, 2 max-pool, 3 + i the
 * output of MLFNBlock i (i = 0 .. 15), 19 s_hat (the 16 blocks' gates, 512), 20 the head row v = 0.5 (x + s) before
 * the L2 normalisation (1024).  For HACNN: 0 input blob (160 x 64), 1 stem, 2 + i x_{i+1}_out (i = 0 .. 2), 5 + i the
 * local map of level i + 1 ([region][h][w][c], 4 regions), 8 theta ([level][region][tx, ty], 24), 9 the head row
 * [fc_global | fc_local] before the normalisations (1024). */
BOXMOT_B200_API int boxmot_b200_reid_debug_stage(void* reid_handle, const float* boxes_xyxy, int n_boxes,
                                                 const uint8_t* image_data, int image_rows, int image_cols,
                                                 int stage, float* out, int out_capacity_floats,
                                                 int* out_floats_per_crop);

#if defined(__cplusplus)
}
#endif
#endif /* BOXMOT_B200_H_ */
