"""ctypes binding of libboxmot_b200.so (the C ABI declared in include/boxmot_b200.h).

There is no CPU fallback: if the library is missing or no CUDA device is visible, every entry point of the
package raises.  Mirrors the role of /root/reference/boxmot/native/trackers/_common.py (ctypes loaders).
"""
from __future__ import annotations

import ctypes
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_void_p
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libboxmot_b200.so"

TRACKER_BYTETRACK = 0
TRACKER_BOTSORT = 1
TRACKER_DEEPOCSORT = 2
TRACKER_STRONGSORT = 3
TRACKER_BOOSTTRACK = 4
TRACKER_OCCLUBOOST = 5
TRACKER_SFSORT = 6


class BoxMOTByteTrackConfig(ctypes.Structure):
    _fields_ = [("min_conf", c_float), ("track_thresh", c_float), ("match_thresh", c_float),
                ("track_buffer", c_int), ("frame_rate", c_int), ("max_obs", c_int)]


class BoxMOTBotSortConfig(ctypes.Structure):
    _fields_ = [("track_high_thresh", c_float), ("track_low_thresh", c_float), ("new_track_thresh", c_float),
                ("track_buffer", c_int), ("match_thresh", c_float), ("proximity_thresh", c_float),
                ("appearance_thresh", c_float), ("cmc_method", c_char_p), ("frame_rate", c_int),
                ("fuse_first_associate", c_int), ("with_reid", c_int), ("max_obs", c_int),
                ("reid_model_path", c_char_p), ("reid_preprocess", c_char_p)]


class BoxMOTB200TrackerConfig(ctypes.Structure):
    _fields_ = [("tracker", c_int), ("n_streams", c_int), ("cap_tracks", c_int), ("cap_dets", c_int),
                ("feat_dim", c_int), ("track_buffer", c_int), ("frame_rate", c_int), ("with_reid", c_int),
                ("fuse_first_associate", c_int), ("removed_stracks_buffer", c_int),
                ("track_high_thresh", c_double), ("track_low_thresh", c_double), ("new_track_thresh", c_double),
                ("match_thresh", c_double), ("second_match_thresh", c_double),
                ("unconfirmed_match_thresh", c_double), ("proximity_thresh", c_double),
                ("appearance_thresh", c_double), ("unconfirmed_emb_scale", c_double),
                ("reid_model_path", c_char_p),
                ("delta_t", c_int), ("max_age", c_int), ("min_hits", c_int), ("embedding_off", c_int),
                ("aw_off", c_int), ("det_thresh", c_double), ("iou_threshold", c_double), ("inertia", c_double),
                ("w_association_emb", c_double), ("alpha_fixed_emb", c_double), ("aw_param", c_double),
                ("q_xy_scaling", c_double), ("q_s_scaling", c_double),
                ("n_init", c_int), ("nn_budget", c_int), ("min_conf", c_double), ("max_cos_dist", c_double),
                ("max_iou_dist", c_double), ("mc_lambda", c_double), ("ema_alpha", c_double),
                ("reid_preprocess", c_int),
                ("use_dlo_boost", c_int), ("use_duo_boost", c_int), ("use_rich_s", c_int), ("use_sb", c_int),
                ("use_vt", c_int), ("s_sim_corr", c_int), ("dlo_boost_coef", c_double), ("lambda_iou", c_double),
                ("lambda_mhd", c_double), ("lambda_shape", c_double), ("min_box_area", c_double),
                ("aspect_ratio_thresh", c_double),
                ("use_second_pass", c_int), ("recovery_max_age", c_int), ("second_pass_max_age", c_int),
                ("second_pass_min_hits", c_int), ("confirm_hits", c_int), ("tentative_max_age", c_int),
                ("ams_enabled", c_int), ("ams_buffer_size", c_int), ("gta_enabled", c_int),
                ("gta_min_track_length", c_int), ("gta_max_gap", c_int), ("lambda_emb_multiplier", c_double),
                ("recovery_appearance_thresh", c_double), ("recovery_iou_thresh", c_double), ("feat_alpha", c_double),
                ("second_iou_thresh", c_double), ("second_appearance_thresh", c_double),
                ("instant_confirm_thresh", c_double), ("duplicate_iou_thresh", c_double), ("ams_alpha0", c_double),
                ("ams_threshold", c_double), ("ams_shrink_ratio", c_double), ("gta_appearance_thresh", c_double),
                ("sf_high_th", c_double), ("sf_match_th_first", c_double), ("sf_new_track_th", c_double),
                ("sf_low_th", c_double), ("sf_match_th_second", c_double), ("sf_dynamic_tuning", c_int),
                ("sf_cth", c_double), ("sf_high_th_m", c_double), ("sf_new_track_th_m", c_double),
                ("sf_match_th_first_m", c_double), ("sf_marginal_timeout", c_int), ("sf_central_timeout", c_int),
                ("sf_frame_width", c_int), ("sf_frame_height", c_int), ("sf_horizontal_margin", c_double),
                ("sf_vertical_margin", c_double), ("sf_log10_table", c_void_p), ("sf_log10_count", c_int)]


class BoxMOTSFSORTConfig(ctypes.Structure):
    _fields_ = [("high_th", c_float), ("match_th_first", c_float), ("new_track_th", c_float), ("low_th", c_float),
                ("match_th_second", c_float), ("dynamic_tuning", c_int), ("cth", c_float), ("high_th_m", c_float),
                ("new_track_th_m", c_float), ("match_th_first_m", c_float), ("obb_theta_damping", c_float),
                ("marginal_timeout", c_int), ("central_timeout", c_int), ("frame_width", c_int), ("frame_height", c_int),
                ("horizontal_margin", c_int), ("vertical_margin", c_int), ("frame_rate", c_int), ("max_obs", c_int)]


# every symbol include/boxmot_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "boxmot_reid_capi_create": (c_int, [c_char_p, c_char_p, POINTER(c_void_p)]),
    "boxmot_reid_capi_destroy": (None, [c_void_p]),
    "boxmot_reid_capi_feature_dim": (c_int, [c_void_p, POINTER(c_int)]),
    "boxmot_reid_capi_compute_features": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int,
                                                  c_void_p, c_int]),
    "boxmot_reid_capi_preprocess": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int]),
    "boxmot_reid_capi_process": (c_int, [c_void_p]),
    "boxmot_reid_capi_postprocess": (c_int, [c_void_p, c_void_p, c_int]),
    "boxmot_reid_capi_last_error": (c_char_p, []),
    "boxmot_bytetrack_create": (c_void_p, [POINTER(BoxMOTByteTrackConfig)]),
    "boxmot_bytetrack_destroy": (None, [c_void_p]),
    "boxmot_bytetrack_reset": (c_int, [c_void_p]),
    "boxmot_bytetrack_update": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int,
                                        c_void_p, c_int, c_int, POINTER(c_int), POINTER(c_int)]),
    "boxmot_bytetrack_last_error": (c_char_p, []),
    "boxmot_botsort_create": (c_void_p, [POINTER(BoxMOTBotSortConfig)]),
    "boxmot_botsort_destroy": (None, [c_void_p]),
    "boxmot_botsort_reset": (c_int, [c_void_p]),
    "boxmot_botsort_update": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p,
                                      c_int, c_int, c_int, c_void_p, c_int, c_int, POINTER(c_int),
                                      POINTER(c_int)]),
    "boxmot_botsort_last_reid_time_ms": (c_int, [c_void_p, POINTER(c_double)]),
    "boxmot_botsort_last_reid_preprocess_time_ms": (c_int, [c_void_p, POINTER(c_double)]),
    "boxmot_botsort_last_reid_process_time_ms": (c_int, [c_void_p, POINTER(c_double)]),
    "boxmot_botsort_last_reid_postprocess_time_ms": (c_int, [c_void_p, POINTER(c_double)]),
    "boxmot_botsort_last_error": (c_char_p, []),
    "boxmot_sfsort_create": (c_void_p, [POINTER(BoxMOTSFSORTConfig)]),
    "boxmot_sfsort_destroy": (None, [c_void_p]),
    "boxmot_sfsort_reset": (c_int, [c_void_p]),
    "boxmot_sfsort_update": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int,
                                     c_void_p, c_int, c_int, POINTER(c_int), POINTER(c_int)]),
    "boxmot_sfsort_last_error": (c_char_p, []),
    "boxmot_b200_tracker_create": (c_void_p, [POINTER(BoxMOTB200TrackerConfig)]),
    "boxmot_b200_tracker_destroy": (None, [c_void_p]),
    "boxmot_b200_tracker_reset": (c_int, [c_void_p]),
    "boxmot_b200_tracker_update_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                 c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_tracker_update_device": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                                  c_int, c_int]),
    "boxmot_b200_tracker_fetch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_tracker_snapshot": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                             POINTER(c_int)]),
    "boxmot_b200_tracker_track_ids": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, POINTER(c_int)]),
    "boxmot_b200_tracker_gta_events": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, POINTER(c_int)]),
    "boxmot_b200_tracker_last_launches": (c_int, [c_void_p, POINTER(c_int)]),
    "boxmot_b200_tracker_last_device_ms": (c_int, [c_void_p, POINTER(c_double), POINTER(c_double)]),
    "boxmot_b200_tracker_set_warp": (c_int, [c_void_p, c_int, c_void_p]),
    "boxmot_b200_tracker_set_cmc": (c_int, [c_void_p, c_char_p]),
    "boxmot_b200_tracker_set_frame_size": (c_int, [c_void_p, c_int, c_int, c_int]),
    "boxmot_b200_cmc_ecc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_double, c_double, c_int, c_void_p, POINTER(c_int),
                                    c_void_p]),
    "boxmot_b200_cmc_sof_create": (c_void_p, [c_double, c_int, c_double, c_double]),
    "boxmot_b200_cmc_sof_apply": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, POINTER(c_int)]),
    "boxmot_b200_cmc_sof_destroy": (None, [c_void_p]),
    "boxmot_b200_tracker_mark": (c_int, [c_void_p, c_int]),
    "boxmot_b200_tracker_elapsed_ms": (c_int, [c_void_p, POINTER(c_double)]),
    "boxmot_b200_tracker_phase_clocks": (c_int, [c_void_p, c_int, c_void_p, c_int]),
    "boxmot_b200_tracker_profile": (c_int, [c_void_p, c_int]),
    "boxmot_b200_tracker_profile_read": (c_int, [c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_last_error": (c_char_p, []),
    "boxmot_b200_jv_dense": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "boxmot_b200_jv_dense_mode": (c_int, [c_int]),
    "boxmot_b200_lsa_solve": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, POINTER(c_int)]),
    "boxmot_b200_lap_solve": (c_int, [c_void_p, c_int, c_int, c_double, c_void_p, c_void_p]),
    "boxmot_b200_kalman_predict": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_int]),
    "boxmot_b200_kalman_update": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_int]),
    "boxmot_b200_kalman_initiate": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_int]),
    "boxmot_b200_iou_cost": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "boxmot_b200_cosine_cost": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "boxmot_b200_pointwise_gemm": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int,
                                           c_void_p, POINTER(c_float)]),
    "boxmot_b200_instance_norm": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                          c_int, c_void_p]),
    "boxmot_b200_resnet_conv": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                        c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                        POINTER(c_float)]),
    "boxmot_b200_vit_layernorm": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_vit_attention": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "boxmot_b200_vit_attention_width": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p]),
    "boxmot_b200_vits_layernorm": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_vits_ain": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_vits_head": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "boxmot_b200_mlfn_group_conv": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                            c_void_p, c_void_p]),
    "boxmot_b200_mlfn_fsm": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                     c_int, c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_f32_pointwise": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                          c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "boxmot_b200_f32_lightconv": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                          c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "boxmot_b200_f32_lightchain": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                           c_int, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "boxmot_b200_f32_gates": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_int, c_int, c_void_p, c_int]),
    "boxmot_b200_f32_head": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int,
                                     c_void_p, c_int, c_int]),
    "boxmot_b200_f32_map": (c_int, [c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                    c_int, c_void_p, c_int]),
    "boxmot_b200_f32_lmbn_head": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                          c_int, c_void_p, c_int, c_int]),
    "boxmot_b200_hacnn_conv": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                       c_void_p, c_void_p, c_int, c_int]),
    "boxmot_b200_hacnn_map": (c_int, [c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p]),
    "boxmot_b200_hacnn_attention": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p]),
    "boxmot_b200_hacnn_stn": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p,
                                      c_int, c_int, c_void_p]),
    "boxmot_b200_hacnn_head": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "boxmot_b200_device_count": (c_int, []),
    "boxmot_b200_reid_debug_stage": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p,
                                             c_int, POINTER(c_int)]),
}

_LIB = None


class B200Error(RuntimeError):
    pass


def load_library():
    """Load the CUDA library; raises (never falls back) when it is missing."""
    global _LIB
    if _LIB is None:
        if not LIB_PATH.exists():
            raise B200Error(
                f"{LIB_PATH} is missing: build it with `python -m boxmot_b200.build` (nvcc, sm_90a). "
                "boxmot_b200 has no CPU fallback.")
        lib = ctypes.CDLL(str(LIB_PATH))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


def require_device():
    lib = load_library()
    if lib.boxmot_b200_device_count() < 1:
        raise B200Error("no CUDA device visible: boxmot_b200 has no CPU fallback")
    return lib


def last_error(lib) -> str:
    msg = lib.boxmot_b200_last_error()
    return msg.decode("utf-8", "replace") if msg else ""
