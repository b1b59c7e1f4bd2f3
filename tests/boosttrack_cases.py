"""BoostTrack golden cases (tests/golden/make_boosttrack_golden.py writes tests/golden/<name>.npz from the unmodified
reference class): name -> (constructor kwargs, frames factory, embeddings factory or None, warps factory or None)."""
from __future__ import annotations

from oracle.streams import bench_stream, stress_stream, unit_embeddings, warp_sequence
from tests.common import mot17_embeddings, mot17_stream

# configs/trackers/boosttrack.yaml (BoostTrack++): what create_tracker("boosttrack") starts from.  use_cmc / cmc_method
# select the estimator, which the golden cases replace by supplied warps (or none)
BOOSTTRACK_YAML = dict(max_age=60, min_hits=3, det_thresh=0.6, iou_threshold=0.3, use_cmc=True, cmc_method="ecc",
                       min_box_area=10, aspect_ratio_thresh=1.6, lambda_iou=0.5, lambda_mhd=0.25, lambda_shape=0.25,
                       use_dlo_boost=True, use_duo_boost=True, dlo_boost_coef=0.65, s_sim_corr=False, use_rich_s=True,
                       use_sb=True, use_vt=True, with_reid=True, adaptive_kf=False)
YAML_NO_CMC = {k: v for k, v in BOOSTTRACK_YAML.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}

CASES = {
    # constructor defaults: DLO + DUO on IoU, no ReID, no rich similarity
    "boosttrack_stress96": ({}, lambda: stress_stream(96, 300), None, None),
    # BoostTrack++ (the YAML): rich similarity, soft BIoU, visual tracklet boost, ReID
    "boosttrackpp_stress96": (YAML_NO_CMC, lambda: stress_stream(96, 300), lambda fr: unit_embeddings(fr, 96, seed=5),
                              None),
    "boosttrack_yaml_stress48_gaps": (YAML_NO_CMC, lambda: stress_stream(48, 200, seed=19, n_classes=3, empty_every=37),
                                      lambda fr: unit_embeddings(fr, 48, seed=5), None),
    # corrected shape similarity with the soft-BIoU boost alone, then the visual-tracklet boost alone
    "boosttrack_scorr_sb_bench128": (dict(use_rich_s=True, s_sim_corr=True, use_sb=True),
                                     lambda: bench_stream(128, 60, hw=(360, 640))[1], None, None),
    "boosttrack_vt_bench128": (dict(use_rich_s=True, use_vt=True, with_reid=True, det_thresh=0.5),
                               lambda: bench_stream(128, 60, hw=(360, 640), stream=3)[1],
                               lambda fr: unit_embeddings(fr, 128, seed=9), None),
    # supplied camera-motion warps every frame (camera_update before the predict step), gaps included
    "boosttrack_warp_stress64": (YAML_NO_CMC, lambda: stress_stream(64, 160, seed=31, empty_every=41),
                                 lambda fr: unit_embeddings(fr, 64, seed=33), lambda: warp_sequence(160, seed=23)),
    # public FRCNN detections of the MOT17-mini fixture, YAML defaults
    "boosttrackpp_yaml_mot17_04": (YAML_NO_CMC, lambda: mot17_stream("04"),
                                   lambda fr: mot17_embeddings("04", fr, seed=11, unit=True), None),
}
SNAP_FRAMES = (1, 2, 10, 50, 150, 299)
