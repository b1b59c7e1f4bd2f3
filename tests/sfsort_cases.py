"""SFSORT golden cases (tests/golden/make_sfsort_golden.py writes tests/golden/<name>.npz from the unmodified reference
class): name -> (constructor kwargs, frames factory, frame size (H, W) of the image passed with every frame)."""
from __future__ import annotations

import numpy as np

from oracle.streams import stress_stream
from tests.common import mot17_stream

# configs/trackers/sfsort.yaml: what create_tracker("sfsort") starts from
SFSORT_YAML = dict(high_th=0.6, match_th_first=0.67, new_track_th=0.7, low_th=0.1, match_th_second=0.3,
                   dynamic_tuning=False, cth=0.5, high_th_m=0.0, new_track_th_m=0.0, match_th_first_m=0.0,
                   marginal_timeout=0, central_timeout=0, horizontal_margin=0, vertical_margin=0)
TIMEOUTS = dict(central_timeout=12, marginal_timeout=4, horizontal_margin=60, vertical_margin=40)
F32_HIGH = float(np.float32(0.6))   # a score equal to high_th's float32 value


def _intermediate_stream():
    """Frames with only intermediate scores (low_th < s < high_th), empty frames, and scores equal to float32(0.6)."""
    frames = stress_stream(48, 160, seed=23)
    rng = np.random.default_rng(5)
    for f, d in enumerate(frames):
        if f % 11 == 10:
            frames[f] = np.zeros((0, 6), np.float32)
        elif f % 7 == 6 and len(d):
            d[:, 4] = rng.uniform(0.15, 0.55, size=len(d)).astype(np.float32)
        elif f % 5 == 3 and len(d):
            d[::4, 4] = np.float32(F32_HIGH)
    return frames


def _dynamic_stream():
    """Dense and sparse frames for the density-tuned thresholds; on every sixth frame exactly one score clears cth, so
    log10(1) = 0 leaves high_th as a float64 0.6 that a float32(0.6) score passes (it would not in float32)."""
    frames = stress_stream(64, 160, seed=41)
    rng = np.random.default_rng(9)
    for f, d in enumerate(frames):
        if f % 6 == 5 and len(d) >= 3:
            d[:, 4] = rng.uniform(0.2, 0.5, size=len(d)).astype(np.float32)
            d[0, 4] = np.float32(0.9)
            d[1::3, 4] = np.float32(F32_HIGH)
    return frames


def _duplicate_stream():
    """Every third frame repeats some detection rows exactly (tied costs in both passes)."""
    frames = stress_stream(32, 120, seed=13)
    for f, d in enumerate(frames):
        if f % 3 == 0 and len(d) >= 2:
            dup = d[::2].copy()
            if f % 2:
                dup[:, 4] = np.float32(0.45)   # the twin of an intermediate-score row
            frames[f] = np.ascontiguousarray(np.concatenate([d, dup], 0))
    return frames


CASES = {
    # constructor defaults: no lost memory (timeouts 0)
    "sfsort_ctor_stress96": ({}, lambda: stress_stream(96, 200), (360, 640)),
    "sfsort_yaml_stress64": (SFSORT_YAML, lambda: stress_stream(64, 200, seed=19, n_classes=3, empty_every=37),
                             (360, 640)),
    # central and marginal timeouts with margins taken from the first image
    "sfsort_timeouts_stress64": (dict(SFSORT_YAML, **TIMEOUTS), lambda: stress_stream(64, 240, seed=31, empty_every=41),
                                 (360, 640)),
    # margins from frame_width / frame_height given to the constructor (differs from the 640 x 360 image)
    "sfsort_framesize_stress64": (dict(TIMEOUTS, frame_width=560, frame_height=300),
                                  lambda: stress_stream(64, 200, seed=37, empty_every=29), (360, 640)),
    "sfsort_dynamic_stress64": (dict(TIMEOUTS, dynamic_tuning=True, cth=0.65, high_th_m=0.05, new_track_th_m=0.04,
                                     match_th_first_m=0.03), _dynamic_stream, (360, 640)),
    "sfsort_intermediate_stress48": (dict(TIMEOUTS, central_timeout=10), _intermediate_stream, (360, 640)),
    "sfsort_duplicates_stress32": (dict(TIMEOUTS), _duplicate_stream, (360, 640)),
    "sfsort_mot17_04": (dict(SFSORT_YAML, central_timeout=30, marginal_timeout=8, horizontal_margin=100,
                             vertical_margin=60), lambda: mot17_stream("04"), (1080, 1920)),
}
