"""Host-side mirror of the reference tracker frontends over the CUDA C ABI.

`ByteTrack` and `BotSort` keep the reference call surface for the per-frame path --
``update(dets, img, embs=None, masks=None) -> TrackResults`` with the input checks of
boxmot/trackers/basetracker.py:120-147,356-372 and the constructor arguments of bytetrack.py:226-257 /
botsort.py:66-118 -- while all track state and arithmetic live on the GPU (csrc/tracker_core.cuh).
This module is tensor plumbing only; there is no CPU implementation behind it.
"""
from __future__ import annotations

import ctypes
from typing import Any, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import B200Error, BoxMOTB200TrackerConfig

# YAML defaults used by the reference's create_tracker (boxmot/configs/trackers/{bytetrack,botsort}.yaml),
# restated as data: this is the configuration contract of the path (SURVEY.md section 2, row 25).
UNBOUNDED_GALLERY_CAP = 1024   # samples per track kept when StrongSORT is built with nn_budget=None

TRACKER_DEFAULTS = {
    "bytetrack": dict(min_conf=0.1, track_thresh=0.6, track_buffer=30, match_thresh=0.9, frame_rate=30),
    "botsort": dict(
        track_high_thresh=0.6296854875023994, track_low_thresh=0.1014392537025336,
        new_track_thresh=0.6246494191492591, track_buffer=40, match_thresh=0.7722224024589055,
        use_cmc=True, cmc_method="sof", frame_rate=30, fuse_first_associate=True, with_reid=True,
        proximity_thresh=0.6084297894561342, appearance_thresh=0.6188818853936099,
        unconfirmed_emb_scale=2.5445206391993294, second_match_thresh=0.28795081514328974,
        unconfirmed_match_thresh=0.41148010638233784, removed_stracks_buffer=329),
    # configs/trackers/deepocsort.yaml: det_thresh 0.5 and w_association_emb 0.75 differ from the constructor defaults
    # (0.3 / 0.5); its `iou_thresh: 0.3` is swallowed by **kwargs in the reference, so iou_threshold keeps its 0.3
    "deepocsort": dict(det_thresh=0.5, max_age=30, min_hits=3, iou_threshold=0.3, delta_t=3, inertia=0.2,
                       w_association_emb=0.75, alpha_fixed_emb=0.95, aw_param=0.5, embedding_off=False,
                       cmc_off=True, aw_off=False, Q_xy_scaling=0.01, Q_s_scaling=0.0001),
    # configs/trackers/ocsort.yaml
    "ocsort": dict(min_conf=0.1, det_thresh=0.6, max_age=30, min_hits=3, delta_t=3, asso_func="iou", use_byte=False,
                   inertia=0.1, Q_xy_scaling=0.01, Q_s_scaling=0.0001),
    "strongsort": dict(min_conf=0.6, ema_alpha=0.9, max_cos_dist=0.4, max_iou_dist=0.7, max_age=30, n_init=3,
                       mc_lambda=0.98, nn_budget=100),
}


class TrackResults(np.ndarray):
    """float32 view over the (M, 8) output rows [x1,y1,x2,y2,id,conf,cls,det_ind] with the named accessors and export
    helpers of the reference class (track_results.py:12-200); AABB layout only (OBB is outside this path)."""

    def __new__(cls, data, masks=None):
        arr = np.asarray(data, dtype=np.float32)
        if arr.ndim == 1 and arr.size > 0:
            arr = arr.reshape(1, -1)
        elif arr.size == 0:
            cols = arr.shape[1] if arr.ndim == 2 else 0
            arr = arr.reshape(0, cols)
        obj = arr.view(cls)
        obj._masks = masks
        return obj

    def __array_finalize__(self, obj):
        self._masks = getattr(obj, "_masks", None)

    @property
    def masks(self):
        return self._masks

    @property
    def is_obb(self) -> bool:
        return self.shape[1] >= 9 if self.ndim == 2 else False

    @property
    def xyxy(self):
        return np.asarray(self[:, :4])

    @property
    def xywh(self):
        boxes = np.asarray(self[:, :4])
        if boxes.size == 0:
            return np.empty((0, 4), dtype=np.float32)
        x1, y1, x2, y2 = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
        return np.stack([(x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1], axis=1)

    @property
    def id(self):
        return np.asarray(self[:, 4]).astype(int)

    @property
    def conf(self):
        return np.asarray(self[:, 5])

    @property
    def cls(self):
        return np.asarray(self[:, 6]).astype(int)

    @property
    def det_ind(self):
        return np.asarray(self[:, 7]).astype(int)

    # ---- export helpers (track_results.py:96-200) ----
    _csv_fields = ["x1", "y1", "x2", "y2", "id", "conf", "cls", "det_ind"]

    def _row(self, i: int):
        return [float(v) for v in self.xyxy[i]] + [int(self.id[i]), float(self.conf[i]), int(self.cls[i]),
                                                   int(self.det_ind[i])]

    def summary(self):
        out = []
        for i in range(len(self)):
            x1, y1, x2, y2 = self.xyxy[i]
            out.append({"id": int(self.id[i]), "conf": float(self.conf[i]), "cls": int(self.cls[i]),
                        "box": {"x1": float(x1), "y1": float(y1), "x2": float(x2), "y2": float(y2)}})
        return out

    def to_json(self, indent=None) -> str:
        import json

        return json.dumps(self.summary(), indent=indent)

    def to_csv(self, frame_id=None) -> str:
        import csv
        import io

        buf = io.StringIO()
        writer = csv.writer(buf)
        for i in range(len(self)):
            writer.writerow(([frame_id] + self._row(i)) if frame_id is not None else self._row(i))
        return buf.getvalue()

    def save_csv(self, path, frame_id=None, header: bool = True) -> None:
        import csv
        from pathlib import Path

        path = Path(path)
        write_header = header and not path.exists()
        path.parent.mkdir(parents=True, exist_ok=True)
        with open(path, "a", newline="") as f:
            if write_header:
                csv.writer(f).writerow((["frame"] + self._csv_fields) if frame_id is not None else self._csv_fields)
            f.write(self.to_csv(frame_id=frame_id))

    def save_mot(self, path, frame_id: int = 0) -> None:
        from pathlib import Path

        path = Path(path)
        path.parent.mkdir(parents=True, exist_ok=True)
        with open(path, "a") as f:
            for i in range(len(self)):
                x1, y1, x2, y2 = self.xyxy[i]
                w, h = x2 - x1, y2 - y1
                f.write(f"{frame_id},{int(self.id[i])},{x1:.2f},{y1:.2f},{w:.2f},{h:.2f},"
                        f"{self.conf[i]:.6f},{int(self.cls[i])},-1\n")


def _check_inputs(dets, img, embs):
    assert isinstance(dets, np.ndarray), (
        f"Unsupported 'dets' input format '{type(dets)}', valid format is np.ndarray")
    assert img is None or isinstance(img, np.ndarray), (
        f"Unsupported 'img_numpy' input format '{type(img)}', valid format is np.ndarray")
    assert len(dets.shape) == 2, "Unsupported 'dets' dimensions, valid number of dimensions is two"
    if embs is not None:
        assert dets.shape[0] == embs.shape[0], "Missmatch between detections and embeddings sizes"
    assert dets.shape[1] == 6, (
        "Unsupported 'dets' 2nd dimension length, valid length is 6 (x1,y1,x2,y2,conf,cls)")


class MultiStreamTracker:
    """`n_streams` independent trackers resident on one GPU, advanced together (one launch sequence/frame).

    Per-stream results equal `n_streams` separate reference trackers (ids start at 1 in every stream)."""

    def __init__(self, tracker: str, n_streams: int = 1, cap_tracks: int = 1024, cap_dets: int = 512,
                 feat_dim: int = 512, reid_blob: Optional[str] = None, reid_preprocess: Optional[str] = None,
                 **params: Any):
        if reid_preprocess not in (None, "resize", "resize_pad"):
            raise ValueError(f"Unknown preprocessing '{reid_preprocess}'. Available: ['resize', 'resize_pad']")
        self.lib = _lib.require_device()
        cfg = BoxMOTB200TrackerConfig()
        kind = tracker.lower()
        if kind == "bytetrack":
            p = dict(min_conf=0.1, track_thresh=0.45, match_thresh=0.8, track_buffer=25, frame_rate=30)
            unknown = set(params) - set(p)
            if unknown:
                raise TypeError(f"unknown ByteTrack parameters: {sorted(unknown)}")
            p.update(params)
            cfg.tracker = _lib.TRACKER_BYTETRACK
            cfg.track_high_thresh = p["track_thresh"]
            cfg.track_low_thresh = p["min_conf"]
            cfg.new_track_thresh = p["track_thresh"]
            cfg.match_thresh = p["match_thresh"]
            cfg.second_match_thresh = 0.5
            cfg.unconfirmed_match_thresh = 0.7
            cfg.removed_stracks_buffer = 0
            cfg.with_reid = 0
            cfg.fuse_first_associate = 1
        elif kind == "botsort":
            p = dict(track_high_thresh=0.5, track_low_thresh=0.1, new_track_thresh=0.6, track_buffer=30,
                     match_thresh=0.8, proximity_thresh=0.5, appearance_thresh=0.25, frame_rate=30,
                     fuse_first_associate=False, with_reid=True, second_match_thresh=0.5,
                     unconfirmed_match_thresh=0.7, unconfirmed_emb_scale=2.0, removed_stracks_buffer=100)
            unknown = set(params) - set(p)
            if unknown:
                raise TypeError(f"unknown BotSort parameters: {sorted(unknown)}")
            p.update(params)
            cfg.tracker = _lib.TRACKER_BOTSORT
            cfg.track_high_thresh = p["track_high_thresh"]
            cfg.track_low_thresh = p["track_low_thresh"]
            cfg.new_track_thresh = p["new_track_thresh"]
            cfg.match_thresh = p["match_thresh"]
            cfg.second_match_thresh = p["second_match_thresh"]
            cfg.unconfirmed_match_thresh = p["unconfirmed_match_thresh"]
            cfg.proximity_thresh = p["proximity_thresh"]
            cfg.appearance_thresh = p["appearance_thresh"]
            cfg.unconfirmed_emb_scale = p["unconfirmed_emb_scale"]
            cfg.removed_stracks_buffer = int(p["removed_stracks_buffer"])
            cfg.with_reid = int(bool(p["with_reid"]))
            cfg.fuse_first_associate = int(bool(p["fuse_first_associate"]))
        elif kind == "deepocsort":
            p = dict(delta_t=3, inertia=0.2, w_association_emb=0.5, alpha_fixed_emb=0.95, aw_param=0.5,
                     embedding_off=False, aw_off=False, Q_xy_scaling=0.01, Q_s_scaling=0.0001, det_thresh=0.3,
                     max_age=30, min_hits=3, iou_threshold=0.3)
            unknown = set(params) - set(p)
            if unknown:
                raise TypeError(f"unknown DeepOcSort parameters: {sorted(unknown)}")
            p.update(params)
            cfg.tracker = _lib.TRACKER_DEEPOCSORT
            cfg.delta_t, cfg.max_age, cfg.min_hits = int(p["delta_t"]), int(p["max_age"]), int(p["min_hits"])
            cfg.embedding_off, cfg.aw_off = int(bool(p["embedding_off"])), int(bool(p["aw_off"]))
            cfg.det_thresh, cfg.iou_threshold, cfg.inertia = p["det_thresh"], p["iou_threshold"], p["inertia"]
            cfg.w_association_emb, cfg.alpha_fixed_emb, cfg.aw_param = p["w_association_emb"], p["alpha_fixed_emb"], p["aw_param"]
            cfg.q_xy_scaling, cfg.q_s_scaling = p["Q_xy_scaling"], p["Q_s_scaling"]
            cfg.with_reid = int(not p["embedding_off"])
            p.setdefault("track_buffer", 0)
            p.setdefault("frame_rate", 30)
            p["track_high_thresh"] = p["det_thresh"]  # detections above det_thresh are embedded
        elif kind == "strongsort":
            p = dict(min_conf=0.1, max_cos_dist=0.2, max_iou_dist=0.7, n_init=3, nn_budget=100, mc_lambda=0.98,
                     ema_alpha=0.9, max_age=30)
            unknown = set(params) - set(p)
            if unknown:
                raise TypeError(f"unknown StrongSort parameters: {sorted(unknown)}")
            p.update(params)
            if p["nn_budget"] is None:
                # the reference keeps every sample of a track for ever (linear_assignment.py:307-331); the device gallery is a
                # ring per track slot, so "unbounded" becomes a large ring: identical until one track has collected more than
                # UNBOUNDED_GALLERY_CAP samples (34 s of uninterrupted matches at 30 fps), after which the oldest is dropped
                import warnings

                warnings.warn(f"StrongSORT nn_budget=None: the device gallery keeps the last {UNBOUNDED_GALLERY_CAP} samples per "
                              "track (the reference's list is unbounded)", stacklevel=3)
                p["nn_budget"] = UNBOUNDED_GALLERY_CAP
            cfg.tracker = _lib.TRACKER_STRONGSORT
            cfg.n_init, cfg.nn_budget, cfg.max_age = int(p["n_init"]), int(p["nn_budget"]), int(p["max_age"])
            cfg.min_conf, cfg.max_cos_dist, cfg.max_iou_dist = p["min_conf"], p["max_cos_dist"], p["max_iou_dist"]
            cfg.mc_lambda, cfg.ema_alpha = p["mc_lambda"], p["ema_alpha"]
            cfg.with_reid = 1
            p.setdefault("track_buffer", 0)
            p.setdefault("frame_rate", 30)
        else:
            raise ValueError(f"tracker '{tracker}' is not part of the B200 hot path "
                             "(bytetrack, botsort, deepocsort, strongsort)")
        cfg.n_streams = int(n_streams)
        cfg.cap_tracks = int(cap_tracks)
        cfg.cap_dets = int(cap_dets)
        if reid_blob:
            # the engine takes the embedding width from the blob: keep this object's stride / width checks in step
            import struct

            with open(reid_blob, "rb") as fh:
                hdr = struct.unpack("<16i", fh.read(64))
            feat_dim = int(hdr[7]) if hdr[7] > 0 else feat_dim
        cfg.feat_dim = int(feat_dim)
        cfg.track_buffer = int(p["track_buffer"])
        cfg.frame_rate = int(p["frame_rate"])
        self._blob = str(reid_blob).encode() if reid_blob else None
        cfg.reid_model_path = self._blob
        cfg.reid_preprocess = 1 if reid_preprocess == "resize_pad" else 0
        self.kind = kind
        self.params = p
        self.n_streams = int(n_streams)
        self.cap_dets = int(cap_dets)
        self.cap_tracks = int(cap_tracks)
        self.feat_dim = int(feat_dim)
        self.with_reid = bool(cfg.with_reid)
        self.has_reid_model = reid_blob is not None
        self.handle = self.lib.boxmot_b200_tracker_create(ctypes.byref(cfg))
        if not self.handle:
            raise B200Error(f"tracker create failed: {_lib.last_error(self.lib)}")
        self.frame_count = 0
        self.cmc = None

    def set_cmc(self, method: Optional[str]) -> None:
        """Camera-motion ESTIMATION on the device from the frames passed to `update`: "ecc" (BoT-SORT, StrongSORT) = the
        reference's ECC estimator with its defaults (motion/cmc/ecc.py:23-108: translation model, eps 1e-5, 100 iterations,
        gray image at scale 0.15), run where the reference runs it (botsort.py:142, strongsort.py:83-86); "sof" (BoT-SORT,
        DeepOCSORT) = the reference's SOF estimator with its defaults (motion/cmc/sof.py; `boxmot_b200.SOF`), run on every
        frame with the detection boxes the reference masks (BoT-SORT: every row, DeepOCSORT: conf > det_thresh); None /
        "none" turns it off (warps are then supplied through `set_warp`).  `reset()` restarts the estimator."""
        m = None if method in (None, "", "none", "None") else str(method)
        if not self.lib.boxmot_b200_tracker_set_cmc(self.handle, m.encode() if m else None):
            raise B200Error(_lib.last_error(self.lib))
        self.cmc = m

    def close(self):
        if getattr(self, "handle", None):
            self.lib.boxmot_b200_tracker_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        if not self.lib.boxmot_b200_tracker_reset(self.handle):
            raise B200Error(_lib.last_error(self.lib))
        self.frame_count = 0

    def set_warp(self, stream: int, warp) -> None:
        """Camera-motion warp (2x3) to apply on the next update of `stream` (BoT-SORT multi_gmc, StrongSORT
        camera_update, DeepOCSORT apply_affine_correction)."""
        w = np.ascontiguousarray(warp, dtype=np.float64).reshape(6)
        if not self.lib.boxmot_b200_tracker_set_warp(self.handle, int(stream), w.ctypes.data):
            raise B200Error(_lib.last_error(self.lib))

    def update(self, dets: Sequence[np.ndarray], imgs: Optional[Sequence[np.ndarray]] = None,
               embs: Optional[Sequence[Optional[np.ndarray]]] = None):
        S = self.n_streams
        assert len(dets) == S, f"expected {S} detection arrays"
        d_arr, d_ptr, rows = [], (ctypes.c_void_p * S)(), (ctypes.c_int * S)()
        for i, d in enumerate(dets):
            d = np.zeros((0, 6), np.float32) if d is None or len(d) == 0 else d
            d = np.ascontiguousarray(d, dtype=np.float32)
            assert d.ndim == 2 and d.shape[1] == 6, (
                "Unsupported 'dets' 2nd dimension length, valid length is 6 (x1,y1,x2,y2,conf,cls)")
            d_arr.append(d)
            d_ptr[i] = d.ctypes.data if len(d) else None
            rows[i] = len(d)
        e_ptr = None
        e_arr = []
        if embs is not None and self.with_reid:
            e_ptr = (ctypes.c_void_p * S)()
            for i, e in enumerate(embs):
                if rows[i] == 0:
                    e_ptr[i] = None
                    continue
                assert e is not None and len(e) == rows[i], "Missmatch between detections and embeddings sizes"
                e = np.ascontiguousarray(e, dtype=np.float32)
                assert e.ndim == 2 and e.shape[1] == self.feat_dim, "embedding width does not match feat_dim"
                e_arr.append(e)
                e_ptr[i] = e.ctypes.data
        i_ptr, ih, iw = None, 0, 0
        i_arr = []
        if (self.with_reid and e_ptr is None) or self.cmc:
            if imgs is None:
                raise B200Error("camera-motion estimation needs the frames" if self.cmc and not (self.with_reid and e_ptr is None)
                                else "BoT-SORT with_reid needs `embs` or frames (and a ReID blob) to embed detections")
            i_ptr = (ctypes.c_void_p * S)()
            for i, im in enumerate(imgs):
                im = np.ascontiguousarray(im, dtype=np.uint8)
                assert im.ndim == 3 and im.shape[2] == 3, "img must be HxWx3 uint8 BGR"
                if i == 0:
                    ih, iw = im.shape[:2]
                assert im.shape[:2] == (ih, iw), "all frames of one batch must share a resolution"
                i_arr.append(im)
                i_ptr[i] = im.ctypes.data
        outs = [np.empty((max(int(rows[i]), 1), 9), np.float32) for i in range(S)]
        o_ptr = (ctypes.c_void_p * S)(*[o.ctypes.data for o in outs])
        o_cap = (ctypes.c_int * S)(*[len(o) for o in outs])
        o_rows = (ctypes.c_int * S)()
        ok = self.lib.boxmot_b200_tracker_update_batch(self.handle, d_ptr, rows, e_ptr, i_ptr, ih, iw, o_ptr, o_cap,
                                                       o_rows)
        if not ok:
            raise B200Error(_lib.last_error(self.lib))
        self.frame_count += 1
        return [TrackResults(outs[i][: o_rows[i], :8].copy()) for i in range(S)]

    # ---- device-resident frame loop (SURVEY 8f-1) ---------------------------------------------------------------
    @staticmethod
    def _dev_ptr(obj, what: str, dtype: str, min_elems: int):
        """Raw device address of a CUDA tensor (`data_ptr()` / `__cuda_array_interface__`) or a plain integer."""
        if obj is None:
            return None
        if isinstance(obj, int):
            return obj
        if hasattr(obj, "data_ptr"):  # torch.Tensor
            if not obj.is_cuda:
                raise B200Error(f"{what} must live in device memory for update_device (got a host tensor)")
            if not obj.is_contiguous():
                raise B200Error(f"{what} must be contiguous")
            if str(obj.dtype).split(".")[-1] != dtype:
                raise B200Error(f"{what} must be {dtype}, got {obj.dtype}")
            if obj.numel() < min_elems:
                raise B200Error(f"{what} holds {obj.numel()} elements, {min_elems} are addressed")
            return int(obj.data_ptr())
        cai = getattr(obj, "__cuda_array_interface__", None)
        if cai is not None:
            if int(np.prod(cai["shape"])) < min_elems:
                raise B200Error(f"{what} is smaller than the {min_elems} elements addressed")
            return int(cai["data"][0])
        raise B200Error(f"{what}: expected a CUDA tensor or a device address")

    def update_device(self, d_dets, det_rows: Sequence[int], d_embs=None, d_images=None,
                      image_hw: Optional[Sequence[int]] = None, sync: bool = True) -> None:
        """Advance every stream by one frame from inputs that already live in HBM (a detector's output boxes and the
        decoded frames): `d_dets` `[n_streams][cap_dets][6]` float32, `d_embs` `[n_streams][cap_dets][feat_dim]`
        float32 or None, `d_images` `[n_streams][H][W][3]` uint8 or None, `det_rows` host ints.  With `sync=False`
        the call returns after enqueueing: ReID of the next frame overlaps this frame's association.  Rows stay on
        the device until `fetch()`."""
        S = self.n_streams
        assert len(det_rows) == S, f"expected {S} detection counts"
        if max(det_rows, default=0) > self.cap_dets:
            raise B200Error(f"{max(det_rows)} detections exceed cap_dets={self.cap_dets}")
        rows = (ctypes.c_int * S)(*[int(r) for r in det_rows])
        ih, iw = (0, 0) if image_hw is None else (int(image_hw[0]), int(image_hw[1]))
        if d_images is not None and image_hw is None:
            shp = tuple(getattr(d_images, "shape", ()))
            if len(shp) < 3:
                raise B200Error("image_hw is required when d_images is a raw address")
            ih, iw = int(shp[-3]), int(shp[-2])
        p_d = self._dev_ptr(d_dets, "d_dets", "float32", S * self.cap_dets * 6)
        p_e = self._dev_ptr(d_embs, "d_embs", "float32", S * self.cap_dets * self.feat_dim)
        p_i = self._dev_ptr(d_images, "d_images", "uint8", S * ih * iw * 3)
        if not self.lib.boxmot_b200_tracker_update_device(self.handle, p_d, rows, p_e, p_i, ih, iw, int(bool(sync))):
            raise B200Error(_lib.last_error(self.lib))
        self.frame_count += 1

    def fetch(self):
        """Rows of the last frame enqueued by `update_device` (waits for the device), one `TrackResults` per stream."""
        S = self.n_streams
        outs = [np.empty((self.cap_dets, 9), np.float32) for _ in range(S)]
        o_ptr = (ctypes.c_void_p * S)(*[o.ctypes.data for o in outs])
        o_cap = (ctypes.c_int * S)(*[self.cap_dets] * S)
        o_rows = (ctypes.c_int * S)()
        if not self.lib.boxmot_b200_tracker_fetch(self.handle, o_ptr, o_cap, o_rows):
            raise B200Error(_lib.last_error(self.lib))
        return [TrackResults(outs[i][: o_rows[i], :8].copy()) for i in range(S)]

    def snapshot(self, stream: int = 0):
        cap = self.cap_tracks
        ids = np.empty(cap, np.int32)
        means = np.empty((cap, 8))
        covs = np.empty((cap, 8, 8))
        n = ctypes.c_int(0)
        ok = self.lib.boxmot_b200_tracker_snapshot(self.handle, stream, ids.ctypes.data, means.ctypes.data,
                                                   covs.ctypes.data, cap, ctypes.byref(n))
        if not ok:
            raise B200Error(_lib.last_error(self.lib))
        return {int(ids[i]): (means[i].copy(), covs[i].copy()) for i in range(n.value)}

    def track_ids(self, which: int, stream: int = 0):
        """Ids of the tracker's list `which` (0 active, 1 lost, 2 removed) in list order."""
        ids = np.empty(max(self.cap_tracks, 1024), np.int32)
        n = ctypes.c_int(0)
        if not self.lib.boxmot_b200_tracker_track_ids(self.handle, stream, int(which), ids.ctypes.data, len(ids), ctypes.byref(n)):
            raise B200Error(_lib.last_error(self.lib))
        return ids[: n.value].tolist()

    def last_launches(self) -> int:
        n = ctypes.c_int(0)
        self.lib.boxmot_b200_tracker_last_launches(self.handle, ctypes.byref(n))
        return n.value

    def last_device_ms(self):
        a, b = ctypes.c_double(0), ctypes.c_double(0)
        self.lib.boxmot_b200_tracker_last_device_ms(self.handle, ctypes.byref(a), ctypes.byref(b))
        return a.value, b.value


class _SingleStreamTracker:
    """BaseTracker-shaped single-stream frontend (basetracker.py:19-147)."""

    _kind = ""
    provides_reid = False
    supports_obb = False

    def __init__(self, per_class: bool = False, cap_tracks: int = 2048, cap_dets: int = 1024,
                 reid_model: Any = None, feat_dim: int = 512, det_thresh: float = 0.3, max_age: int = 30,
                 max_obs: int = 50, min_hits: int = 3, iou_threshold: float = 0.3, nr_classes: int = 80,
                 asso_func: str = "iou", is_obb: bool = False, **params: Any):
        if per_class:
            raise NotImplementedError("per_class=True is out of scope for the B200 hot path (SURVEY N15)")
        if is_obb:
            raise NotImplementedError("OBB detections are out of scope for the B200 hot path")
        if asso_func != "iou":
            raise NotImplementedError("only asso_func='iou' is implemented")
        self.per_class = False
        self.det_thresh, self.max_age, self.max_obs, self.min_hits = det_thresh, max_age, max_obs, min_hits
        self.iou_threshold, self.nr_classes, self.is_obb = iou_threshold, nr_classes, False
        self.model = reid_model
        blob = getattr(reid_model, "blob_path", None)
        if reid_model is not None and blob is not None:
            feat_dim = int(getattr(reid_model, "feature_dim", feat_dim))
        if self._kind == "deepocsort" and max_obs < max_age + 4:
            # the reference's un-freeze replay looks its pre-gap anchor up in a history deque of max_obs entries
            # (xysr.py:384-399) and silently skips the replay once a gap has pushed it out; the device keeps the anchor
            raise NotImplementedError("DeepOCSORT needs max_obs >= max_age + 4 (history window of the un-freeze replay)")
        if self._kind == "deepocsort":  # BaseTracker settings that DeepOCSORT's update actually reads
            params = dict(params, det_thresh=det_thresh, max_age=max_age, min_hits=min_hits, iou_threshold=iou_threshold)
        if self._kind == "strongsort":  # Tracker(max_age=self.max_age) (strongsort.py:56-64)
            params = dict(params, max_age=max_age)
        self._engine = MultiStreamTracker(self._kind, 1, cap_tracks, cap_dets, feat_dim, reid_blob=blob,
                                          reid_preprocess=getattr(reid_model, "preprocess_name", None) if blob else None, **params)
        self.provides_reid = blob is not None
        self.with_reid = self._engine.with_reid
        self.frame_count = 0

    def reset(self):
        self._engine.reset()
        self.frame_count = 0

    def set_cmc(self, method: Optional[str]) -> None:
        """Turn on-device camera-motion estimation on or off after construction (`MultiStreamTracker.set_cmc`):
        "sof" for BoT-SORT and DeepOCSORT, "ecc" for BoT-SORT and StrongSORT, None to turn it off."""
        self._engine.set_cmc(method)

    def update(self, dets, img=None, embs=None, masks=None, warp=None) -> TrackResults:
        """`warp`: optional 2x3 camera-motion matrix for this frame (BoT-SORT, DeepOCSORT, StrongSORT); the reference
        estimates it with OpenCV inside update() (botsort.py:142-144, deepocsort.py:345-348, strongsort.py:83-86), here the
        caller supplies it."""
        if warp is not None:
            self._engine.set_warp(0, warp)
        if hasattr(dets, "data") and not isinstance(dets, np.ndarray):
            dets = dets.data
        if isinstance(dets, memoryview):
            dets = np.array(dets, dtype=np.float32)
        if dets is None or len(dets) == 0:
            dets = np.empty((0, 6), dtype=np.float32)
            embs = None if embs is None or len(embs) else embs
        _check_inputs(dets, img, embs)
        eng = self._engine
        if eng.with_reid and embs is None and not eng.has_reid_model:
            # foreign ReID backend (any object with get_features): embed the first-round detections on its
            # own device and hand the rows to the tracker, exactly where botsort.py:191-192 calls the model
            if self.model is None:
                raise B200Error("with_reid=True needs reid_model=, embs=, or with_reid=False")
            # the device re-derives the split from the float32 rows it receives: decide on the same rounded values
            conf = np.asarray(dets, dtype=np.float32)[:, 4].astype(np.float64)
            first = conf >= eng.params["min_conf"] if eng.kind == "strongsort" else conf > eng.params["track_high_thresh"]
            embs = np.zeros((len(dets), eng.feat_dim), np.float32)
            if first.any():
                embs[first] = np.asarray(self.model.get_features(dets[first][:, :4], img), dtype=np.float32)
        out = eng.update([dets], None if img is None else [img], None if embs is None else [embs])[0]
        self.frame_count = eng.frame_count
        return out

    def snapshot(self):
        return self._engine.snapshot(0)

    # ---- attributes the reference's callers read (basetracker.py:76, 374-390) --------------------------------------
    class TrackView:
        """Read-only view of one live track: `id`, Kalman `mean` / `covariance` (float64 copies of the device state)."""

        __slots__ = ("id", "mean", "covariance")

        def __init__(self, tid, mean, cov):
            self.id, self.mean, self.covariance = tid, mean, cov

    def _views(self, which):
        state = self._engine.snapshot(0)
        return [self.TrackView(k, *state.get(k, (None, None))) for k in self._engine.track_ids(which)]

    @property
    def active_tracks(self):
        """The tracker's active list, in list order, as views of the device-resident state (one synchronising snapshot
        per access).  basetracker.py:386."""
        return self._views(0)

    @property
    def lost_stracks(self):
        """Lost tracks in list order (BoT-SORT / ByteTrack; the other trackers keep none).  basetracker.py:389."""
        return self._views(1)

    @property
    def removed_stracks(self):
        """Removed tracks: ids only (their Kalman state is gone).  BoT-SORT: the deque of `removed_stracks_buffer` ids,
        oldest first; ByteTrack: every removed id, in slot order.  basetracker.py:390."""
        return self._views(2)

    def get_active_tracks_for_display(self) -> list:
        return list(self.active_tracks)


class ByteTrack(_SingleStreamTracker):
    """ByteTrack on the GPU; arguments as boxmot/trackers/bbox/bytetrack/bytetrack.py:226-257."""

    _kind = "bytetrack"

    def __init__(self, min_conf: float = 0.1, track_thresh: float = 0.45, match_thresh: float = 0.8,
                 track_buffer: int = 25, frame_rate: int = 30, **kwargs: Any):
        super().__init__(min_conf=min_conf, track_thresh=track_thresh, match_thresh=match_thresh,
                         track_buffer=track_buffer, frame_rate=frame_rate, **kwargs)


class BotSort(_SingleStreamTracker):
    """BoT-SORT on the GPU; arguments as boxmot/trackers/bbox/botsort/botsort.py:66-118.

    `use_cmc=True` with `cmc_method="ecc"` (the reference constructor's method) estimates the camera warp on the device
    every frame from `img` (SURVEY 8f-3, `MultiStreamTracker.set_cmc`).  SOF (botsort.yaml's method) also runs on the
    device: build with `use_cmc=False` and call `set_cmc("sof")`.  ORB and SIFT are outside this path: pass their warp
    through `update(..., warp=)`.  `use_cmc` defaults to False here (the reference: True)."""

    _kind = "botsort"

    def __init__(self, reid_model: Any = None, track_high_thresh: float = 0.5, track_low_thresh: float = 0.1,
                 new_track_thresh: float = 0.6, track_buffer: int = 30, match_thresh: float = 0.8,
                 proximity_thresh: float = 0.5, appearance_thresh: float = 0.25, use_cmc: bool = False,
                 cmc_method: str = "ecc", frame_rate: int = 30, fuse_first_associate: bool = False,
                 with_reid: bool = True, second_match_thresh: float = 0.5,
                 unconfirmed_match_thresh: float = 0.7, unconfirmed_emb_scale: float = 2.0,
                 removed_stracks_buffer: int = 100, **kwargs: Any):
        if use_cmc and cmc_method != "ecc":
            raise NotImplementedError(f"use_cmc=True with cmc_method='{cmc_method}': only 'ecc' is estimated on the device "
                                      "(pass use_cmc=False and supply the warp through update(..., warp=))")
        super().__init__(reid_model=reid_model if with_reid else None, track_high_thresh=track_high_thresh,
                         track_low_thresh=track_low_thresh, new_track_thresh=new_track_thresh,
                         track_buffer=track_buffer, match_thresh=match_thresh, proximity_thresh=proximity_thresh,
                         appearance_thresh=appearance_thresh, frame_rate=frame_rate,
                         fuse_first_associate=fuse_first_associate, with_reid=with_reid,
                         second_match_thresh=second_match_thresh,
                         unconfirmed_match_thresh=unconfirmed_match_thresh,
                         unconfirmed_emb_scale=unconfirmed_emb_scale,
                         removed_stracks_buffer=removed_stracks_buffer, **kwargs)
        if use_cmc:
            self._engine.set_cmc("ecc")


class DeepOcSort(_SingleStreamTracker):
    """DeepOCSORT on the GPU; arguments as boxmot/trackers/bbox/deepocsort/deepocsort.py:263-300.  `cmc_off=False` runs
    the reference's SOF estimator on the device on every frame, from `img` and the detections with conf > det_thresh
    (deepocsort.py:330-349).  With the default `cmc_off=True` (the reference: False) a warp obtained elsewhere is
    applied exactly as the reference applies its own (`apply_affine_correction` on every track before the predict
    step) when passed as `update(dets, img, embs, warp=warp_2x3)`."""

    _kind = "deepocsort"

    def __init__(self, reid_model: Any = None, delta_t: int = 3, inertia: float = 0.2, w_association_emb: float = 0.5,
                 alpha_fixed_emb: float = 0.95, aw_param: float = 0.5, embedding_off: bool = False,
                 cmc_off: bool = True, aw_off: bool = False, Q_xy_scaling: float = 0.01, Q_s_scaling: float = 0.0001,
                 det_thresh: float = 0.3, max_age: int = 30, min_hits: int = 3, iou_threshold: float = 0.3,
                 **kwargs: Any):
        super().__init__(reid_model=None if embedding_off else reid_model, delta_t=delta_t, inertia=inertia,
                         w_association_emb=w_association_emb, alpha_fixed_emb=alpha_fixed_emb, aw_param=aw_param,
                         embedding_off=embedding_off, aw_off=aw_off, Q_xy_scaling=Q_xy_scaling,
                         Q_s_scaling=Q_s_scaling, det_thresh=det_thresh, max_age=max_age, min_hits=min_hits,
                         iou_threshold=iou_threshold, **kwargs)
        if not cmc_off:
            self._engine.set_cmc("sof")


class OcSort(_SingleStreamTracker):
    """OC-SORT on the GPU; arguments as boxmot/trackers/bbox/ocsort/ocsort.py:331-362.  For axis-aligned boxes the
    reference class is the DeepOCSORT update with the appearance and camera-motion terms removed (same XYSR filter, same
    `associate()`, same observation-centric second round), so it runs on the DeepOCSORT device core with the embedding
    term off; ids / rows are pinned on goldens from the unmodified OcSort class.  `use_byte=True` (an extra ByteTrack-style
    round on low-confidence detections) is not implemented; `min_conf` only feeds that round."""

    _kind = "deepocsort"

    def __init__(self, min_conf: float = 0.1, delta_t: int = 3, inertia: float = 0.2, use_byte: bool = False,
                 Q_xy_scaling: float = 0.01, Q_s_scaling: float = 0.0001, **kwargs: Any):
        if use_byte:
            raise NotImplementedError("use_byte=True (BYTE second association) is not implemented on the B200 path")
        kwargs.pop("reid_model", None)
        self.min_conf, self.use_byte = min_conf, False
        super().__init__(reid_model=None, delta_t=delta_t, inertia=inertia, embedding_off=True, aw_off=True,
                         Q_xy_scaling=Q_xy_scaling, Q_s_scaling=Q_s_scaling, **kwargs)

    def update(self, dets, img=None, embs=None, masks=None, warp=None) -> TrackResults:
        return super().update(dets, img, None, masks)


class StrongSort(_SingleStreamTracker):
    """StrongSORT on the GPU; arguments as boxmot/trackers/bbox/strongsort/strongsort.py:38-67 (`max_age` is the
    BaseTracker setting the reference forwards to its Tracker).  The reference estimates a camera warp with ECC on
    every frame that has tracks (strongsort.py:67,83-86): `cmc="ecc"` does the same on the device from `img`
    (SURVEY 8f-3); with the default `cmc=None` the warp is an input (`update(..., warp=)`, identity when omitted).
    `camera_update` itself always runs, as in the reference (SURVEY N6)."""

    _kind = "strongsort"

    def __init__(self, reid_model: Any = None, min_conf: float = 0.1, max_cos_dist: float = 0.2,
                 max_iou_dist: float = 0.7, n_init: int = 3, nn_budget: int = 100, mc_lambda: float = 0.98,
                 ema_alpha: float = 0.9, cmc: Optional[str] = None, **kwargs: Any):
        if cmc not in (None, "", "none", "ecc"):
            raise NotImplementedError(f"cmc='{cmc}': StrongSORT's estimator is 'ecc' (or None: supplied warps)")
        super().__init__(reid_model=reid_model, min_conf=min_conf, max_cos_dist=max_cos_dist,
                         max_iou_dist=max_iou_dist, n_init=n_init, nn_budget=nn_budget, mc_lambda=mc_lambda,
                         ema_alpha=ema_alpha, **kwargs)
        if cmc == "ecc":
            self._engine.set_cmc("ecc")


def _flatten_yaml_defaults(node, acc=None):
    """`<param>: {default: ...}` entries of a reference tracker YAML, nested conditional parameters included
    (what `flatten_yaml_config` + `details["default"]` produce in tracker_zoo.py:112-119)."""
    acc = {} if acc is None else acc
    if isinstance(node, dict):
        for k, v in node.items():
            if isinstance(v, dict) and "default" in v:
                acc[str(k)] = v["default"]
            _flatten_yaml_defaults(v, acc)
    elif isinstance(node, list):
        for v in node:
            _flatten_yaml_defaults(v, acc)
    return acc


_CMC_WARNED: dict = {}


def resolve_tracker_args(tracker_type, tracker_config=None, evolve_param_dict=None, overrides=None):
    """(kind, class, constructor kwargs) exactly as the reference's `create_tracker` would assemble them
    (tracker_zoo.py:103-147): `evolve_param_dict` replaces the YAML defaults wholesale, `tracker_config` is a YAML file
    in the reference's format (default: the built-in copy of configs/trackers/<kind>.yaml), keys the reference's
    constructors swallow in **kwargs are dropped.  Camera-motion estimation is outside this path: `use_cmc` is forced
    off / `cmc_off` on whatever the configuration says.  No GPU is touched here."""
    import inspect

    kind = str(tracker_type).lower()
    classes = {"bytetrack": ByteTrack, "botsort": BotSort, "deepocsort": DeepOcSort, "strongsort": StrongSort, "ocsort": OcSort}
    if kind not in classes:
        raise ValueError(f"Unknown tracker type: '{tracker_type}'. Available trackers are: {', '.join(classes)} "
                         "(the trackers that are part of the B200 hot path)")
    if evolve_param_dict is not None:
        args = dict(evolve_param_dict)
    elif tracker_config is not None:
        import yaml

        with open(tracker_config, "r", encoding="utf-8") as f:
            args = _flatten_yaml_defaults(yaml.safe_load(f) or {})
    else:
        args = dict(TRACKER_DEFAULTS[kind])
    args.update(overrides or {})
    cls = classes[kind]
    accepted = set(inspect.signature(cls.__init__).parameters) | set(
        inspect.signature(_SingleStreamTracker.__init__).parameters) | {"cap_tracks", "cap_dets", "feat_dim"}
    accepted -= {"self", "params", "kwargs"}
    args = {k: v for k, v in args.items() if k in accepted}   # the reference's **kwargs swallows the rest
    # Camera-motion estimation: ECC runs on the device (StrongSORT always uses it in the reference; BoT-SORT when
    # cmc_method is "ecc").  The feature-based estimators (sof -- botsort.yaml's and DeepOCSORT's default --, orb, sift) are
    # OpenCV pipelines outside the path: there the estimator is replaced by a warp the caller supplies through
    # update(..., warp=).  Say so once instead of diverging silently.
    method = args.get("cmc_method", "ecc")
    bot_ecc = kind == "botsort" and bool(args.get("use_cmc", False)) and method == "ecc"
    wants_cmc = (kind == "botsort" and args.get("use_cmc", False) and not bot_ecc) or \
        (kind == "deepocsort" and not args.get("cmc_off", False))
    if wants_cmc and not _CMC_WARNED.get(kind):
        import warnings

        _CMC_WARNED[kind] = True
        warnings.warn(f"boxmot_b200.create_tracker('{kind}'): the reference configuration runs camera-motion compensation "
                      f"({method if kind == 'botsort' else 'sof'}); this tracker is built with it off and applies a warp supplied "
                      "through update(..., warp=), without one it behaves as with CMC off -- call tracker.set_cmc('sof') "
                      "(BoT-SORT, DeepOCSORT) to estimate SOF on the device like the reference", stacklevel=3)
    args.pop("cmc_method", None)
    if kind == "botsort":
        args["use_cmc"] = bot_ecc
        if bot_ecc:
            args["cmc_method"] = "ecc"
    if kind == "deepocsort":
        args["cmc_off"] = True
    if kind == "strongsort":
        args.setdefault("cmc", "ecc")   # strongsort.py:67: always ECC
    args.pop("per_class", None)
    return kind, cls, args


def create_tracker(tracker_type, tracker_config=None, reid_weights=None, device=None, half=None, per_class=None,
                   evolve_param_dict=None, reid_preprocess=None, reid_model: Any = None, tracker_backend: str = "python",
                   **overrides: Any):
    """Same signature and argument meaning as boxmot/trackers/tracker_zoo.py:33-147 (positional callers included) for
    the four trackers of the path; `tracker_backend` "python" and "cpp" both resolve to this library.

    `reid_weights` may be a `.pt` state dict or a `.b200reid` blob; it is converted once and loaded on the GPU.
    `**overrides` (an extension) are applied on top of the configuration.  CMC is always off (see BotSort)."""
    kind, cls, args = resolve_tracker_args(tracker_type, tracker_config, evolve_param_dict, overrides)
    per_class = bool(per_class)
    if kind in ("bytetrack", "ocsort"):   # motion-only trackers: no ReID backend (tracker_zoo.py:124-130)
        return cls(per_class=per_class, **args)
    wants_reid = args.get("with_reid", True) and not args.get("embedding_off", False)
    if reid_model is None and reid_weights is not None and wants_reid:
        from .reid import B200ReID

        reid_model = B200ReID(reid_weights, device=device, half=bool(half), preprocess=reid_preprocess)
    tracker = cls(reid_model=reid_model, per_class=per_class, **args)
    # the reference warms the backend up here (tracker_zoo.py:145-146); a B200ReID has nothing lazy to warm
    if getattr(tracker, "model", None) is not None and not tracker.provides_reid and hasattr(tracker.model, "warmup"):
        tracker.model.warmup()
    return tracker
