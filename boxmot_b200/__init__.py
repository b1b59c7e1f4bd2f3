"""boxmot_b200 -- H100-native (sm_90a CUDA) drop-in for BoxMOT's per-frame track-update hot path.

Public surface mirrors the reference seams for this path only (SURVEY.md section 8b):
  * ``ByteTrack`` / ``BotSort`` / ``DeepOcSort`` / ``OcSort`` / ``StrongSort`` / ``BoostTrack`` / ``OccluBoost`` / ``SFSORT``: ``update(dets, img, embs=None) -> TrackResults`` like
    boxmot/trackers/basetracker.py:120-147, backed by the C ABI in include/boxmot_b200.h.
  * ``B200ReID`` (boxmot_b200.reid): ``get_features(xyxys, img)`` + the staged quartet of
    boxmot/reid/backends/base_backend.py:148-244.
  * ``MultiStreamTracker``: S independent trackers advanced by one launch sequence per frame.
  * ``SOF`` (boxmot_b200.cmc): the reference's sparse-optical-flow camera-motion estimator, ``apply(img, dets)``.
Nothing here falls back to the CPU; the CUDA library must be present and a GPU visible.
"""
from ._lib import B200Error, load_library, require_device  # noqa: F401
from .cmc import SOF  # noqa: F401
from .trackers import (BoostTrack, BotSort, ByteTrack, DeepOcSort, MultiStreamTracker, OccluBoost, OcSort, SFSORT, StrongSort,  # noqa: F401
                       TrackResults,  # noqa: F401
                       create_tracker)  # noqa: F401

__all__ = ["ByteTrack", "BotSort", "DeepOcSort", "OcSort", "StrongSort", "BoostTrack", "OccluBoost", "SFSORT", "MultiStreamTracker", "TrackResults", "SOF", "create_tracker", "B200Error",
           "load_library", "require_device"]
