"""OccluBoost golden cases (tests/golden/make_occluboost_golden.py writes tests/golden/<name>.npz from the unmodified
reference class): name -> (constructor kwargs, frames factory, embeddings factory or None, warps factory or None)."""
from __future__ import annotations

import numpy as np

from oracle.streams import stress_stream, unit_embeddings, warp_sequence
from tests.common import mot17_embeddings, mot17_stream

# configs/trackers/occluboost.yaml: what create_tracker("occluboost") starts from.  use_cmc / cmc_method select the
# estimator, which the golden cases replace by supplied warps (or none)
OCCLUBOOST_YAML = dict(
    max_age=146, min_hits=1, det_thresh=0.5678626013369781, iou_threshold=0.2957128153631725, use_cmc=True,
    cmc_method="sof", min_box_area=73, aspect_ratio_thresh=1.4888137942764672, lambda_iou=1.0784558316374715,
    lambda_mhd=0.304435887183232, lambda_shape=1.6709449476805447, use_dlo_boost=True, dlo_boost_coef=1.2061962091907352,
    use_duo_boost=False, s_sim_corr=False, use_rich_s=False, use_sb=True, use_vt=True, with_reid=True,
    recovery_appearance_thresh=0.6732855110134396, recovery_iou_thresh=0.24380051350243462, recovery_max_age=113,
    feat_alpha=0.8324072665785186, track_low_thresh=0.04473431588067598, use_second_pass=True,
    second_iou_thresh=0.8131671757478834, second_appearance_thresh=0.364089272226479, second_pass_max_age=8,
    second_pass_min_hits=7, new_track_thresh=0.7128242784621849, confirm_hits=2,
    instant_confirm_thresh=0.6783889178413256, tentative_max_age=3, duplicate_iou_thresh=0.9571823233925608,
    ams_enabled=True, ams_alpha0=0.8732388616784778, ams_threshold=0.9206232808452425, ams_buffer_size=57,
    ams_shrink_ratio=0.6934881647679682, lambda_emb_multiplier=2.9476295884842885, gta_enabled=False,
    gta_appearance_thresh=0.7125445489563044, gta_min_track_length=7, gta_smooth_tau=14.757519908748044,
    gta_interpolate=False, gta_max_gap=40, adaptive_kf=False)
YAML_NO_CMC = {k: v for k, v in OCCLUBOOST_YAML.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}


def gta_stream(n_objects=24, n_frames=240, seed=41, dim=128, hw=(360, 640)):
    """Objects on straight paths that vanish for 10-50 frames and come back with the same appearance (a prototype per
    identity plus small noise, unit rows): the stream the graveyard resurrection needs.  Returns (frames, embeddings)."""
    h, w = hw
    rng = np.random.default_rng(seed)
    cx, cy = rng.uniform(60, w - 60, n_objects), rng.uniform(60, h - 60, n_objects)
    vx, vy = rng.normal(0, 1.5, n_objects), rng.normal(0, 1.0, n_objects)
    bw, bh = rng.uniform(25, 50, n_objects), rng.uniform(60, 100, n_objects)
    proto = rng.normal(size=(n_objects, dim)).astype(np.float32)
    gone = np.zeros((n_objects, n_frames), bool)
    for k in range(n_objects):
        t = int(rng.integers(15, 60))
        while t < n_frames:
            g = int(rng.integers(10, 51))
            gone[k, t:t + g] = True
            t += g + int(rng.integers(30, 80))
    frames, embs = [], []
    for f in range(n_frames):
        cx += vx
        cy += vy
        vx[(cx < 40) | (cx > w - 40)] *= -1
        vy[(cy < 50) | (cy > h - 50)] *= -1
        idx = np.nonzero(~gone[:, f] & (rng.random(n_objects) >= 0.05))[0]
        j = rng.normal(0, 1.0, (idx.size, 2))
        d = np.stack([cx[idx] + j[:, 0] - bw[idx] / 2, cy[idx] + j[:, 1] - bh[idx] / 2, cx[idx] + j[:, 0] + bw[idx] / 2,
                      cy[idx] + j[:, 1] + bh[idx] / 2, rng.uniform(0.3, 0.95, idx.size), np.zeros(idx.size)], 1)
        e = proto[idx] + 0.3 * rng.normal(size=(idx.size, dim)).astype(np.float32)
        e = e / np.linalg.norm(e, axis=1, keepdims=True) if idx.size else e
        frames.append(d.astype(np.float32).reshape(-1, 6))
        embs.append(np.asarray(e, np.float32).reshape(-1, dim))
    return frames, embs


CASES = {
    # constructor defaults with ReID: GTA on, second pass off
    "occluboost_ctor_stress96": (dict(with_reid=True), lambda: stress_stream(96, 300),
                                 lambda fr: unit_embeddings(fr, 96, seed=5), None),
    # the YAML without CMC: second pass on, GTA off
    "occluboost_yaml_stress96": (YAML_NO_CMC, lambda: stress_stream(96, 300, seed=3),
                                 lambda fr: unit_embeddings(fr, 96, seed=7), None),
    # no ReID: the second pass without the appearance gate, no recovery, no GTA
    "occluboost_noreid_stress64": (dict(YAML_NO_CMC, with_reid=False), lambda: stress_stream(64, 200, seed=13), None,
                                   None),
    # supplied camera-motion warps every frame
    "occluboost_warp_stress64": (dict(YAML_NO_CMC, gta_enabled=True), lambda: stress_stream(64, 160, seed=31, empty_every=41),
                                 lambda fr: unit_embeddings(fr, 64, seed=33), lambda: warp_sequence(160, seed=23)),
    # empty frames and three classes
    "occluboost_gaps_stress48": (dict(with_reid=True, use_second_pass=True),
                                 lambda: stress_stream(48, 200, seed=19, n_classes=3, empty_every=37),
                                 lambda fr: unit_embeddings(fr, 48, seed=5), None),
    # public FRCNN detections of the MOT17-mini fixture, YAML defaults
    "occluboost_yaml_mot17_04": (YAML_NO_CMC, lambda: mot17_stream("04"),
                                 lambda fr: mot17_embeddings("04", fr, seed=11, unit=True), None),
    # identities absent for 10-50 frames: burial, resurrection with interpolated gap rows, smoothing
    "occluboost_gta24": (dict(with_reid=True, max_age=5, min_hits=2, gta_min_track_length=3, gta_appearance_thresh=0.6,
                              gta_max_gap=60), lambda: gta_stream()[0], lambda fr: gta_stream()[1], None),
    # branch forcing: duplicates, tentative expiry, damped AMS updates, second pass on young tracks
    "occluboost_branches_stress96": (dict(with_reid=True, duplicate_iou_thresh=0.3, confirm_hits=3, tentative_max_age=0,
                                          ams_threshold=0.05, ams_shrink_ratio=1.0, use_second_pass=True,
                                          second_pass_min_hits=1, second_iou_thresh=0.3, second_appearance_thresh=0.0,
                                          recovery_appearance_thresh=0.6, recovery_max_age=5, new_track_thresh=0.4,
                                          instant_confirm_thresh=0.8),
                                     lambda: stress_stream(96, 200, seed=57), lambda fr: unit_embeddings(fr, 96, seed=9),
                                     None),
}
SNAP_FRAMES = (1, 2, 10, 50, 150, 299)
