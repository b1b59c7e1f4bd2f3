"""`B200ReID`: the reference's ReID backend contract over the CUDA C ABI.

Mirrors boxmot/reid/backends/base_backend.py:148-244 (`get_features(xyxys, img)` returning L2-normalised
float32 rows, the staged `get_crops / inference_preprocess / forward / inference_postprocess` quartet the
timing wrappers call, `warmup()`, and the attributes `device, half, input_shape, nhwc, mean_array, std_array`)
and boxmot/native/reid/capi.py:346-507 (the ctypes adapter over `boxmot_reid_capi_*`).
All arithmetic runs in libboxmot_b200.so on the GPU; this file only moves buffers.
"""
from __future__ import annotations

import ctypes
from pathlib import Path
from typing import Optional

import numpy as np

from . import _lib
from ._lib import B200Error
from .weights import ARCH_CLIP, ARCH_HACNN, ARCH_LMBN_N, ARCH_VIT, export_blob, read_blob


class _StagedCrops:
    """Opaque token returned by get_crops(): the crops already live in the handle on the device."""

    def __init__(self, n: int):
        self.n = n

    def __len__(self):
        return self.n


class B200ReID:
    input_shape = (256, 128)
    nhwc = True
    mean_array = np.array([0.485, 0.456, 0.406], dtype=np.float32)
    std_array = np.array([0.229, 0.224, 0.225], dtype=np.float32)

    def __init__(self, weights, device=None, half: bool = False, preprocess: Optional[str] = None):
        if preprocess not in (None, "resize", "resize_pad"):
            raise ValueError(f"Unknown preprocessing '{preprocess}'. Available: ['resize', 'resize_pad']")   # preprocessing.py:56-62
        self.preprocess_name = preprocess or "resize"   # DEFAULT_PREPROCESS of the reference's Python loaders
        # half=True is accepted for interface compatibility (the reference's call sites pass it): the network still runs
        # in float32 on the device -- at least the reference's precision -- and the rows handed back to the caller are
        # rounded to float16, the dtype the reference returns in that mode.  Inside a tracker the embeddings never leave
        # the device and stay float32 either way.
        self.lib = _lib.require_device()
        self.blob_path = str(export_blob(weights)) if isinstance(weights, (str, Path)) else None
        if self.blob_path is None:
            raise TypeError("weights must be a path to a .pt checkpoint or a .b200reid blob")
        header, _ = read_blob(self.blob_path)
        self.feature_dim = int(header[7])
        if header[2] == ARCH_LMBN_N:
            self.input_shape = (int(header[9]), 128)   # LMBN_n runs on 384x128 crops (base_backend.py:59-60)
        if header[2] == ARCH_HACNN:
            self.input_shape = (int(header[9]), int(header[10]))   # HACNN runs on 160x64 crops (base_backend.py:61-62)
        if header[2] == ARCH_VIT:
            self.input_shape = (int(header[9]), int(header[10]))   # vit_tiny*: 384x128, vit_nano*: 256x128 (base_backend.py:59-64)
        if header[2] == ARCH_CLIP:
            # CLIP: 256x128, or 256x256 for the vehicle models; mean = std = 0.5 (base_backend.py:52-58)
            self.input_shape = (int(header[9]), int(header[10]))
            self.mean_array = np.array([0.5, 0.5, 0.5], dtype=np.float32)
            self.std_array = np.array([0.5, 0.5, 0.5], dtype=np.float32)
        self.half = bool(half)
        self.device = "cuda:0"
        self.handle = ctypes.c_void_p()
        ok = self.lib.boxmot_reid_capi_create(self.blob_path.encode(), self.preprocess_name.encode(), ctypes.byref(self.handle))
        if not ok:
            raise B200Error(f"boxmot_reid_capi_create failed: {self._err()}")
        dim = ctypes.c_int(0)
        self.lib.boxmot_reid_capi_feature_dim(self.handle, ctypes.byref(dim))
        assert dim.value == self.feature_dim

    def _err(self) -> str:
        m = self.lib.boxmot_reid_capi_last_error()
        return m.decode("utf-8", "replace") if m else ""

    def close(self):
        if getattr(self, "handle", None):
            self.lib.boxmot_reid_capi_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _boxes(xyxys) -> np.ndarray:
        b = np.asarray(xyxys, dtype=np.float32)
        if b.size == 0:
            return b.reshape(0, 4)
        if b.ndim == 1:
            b = b.reshape(1, -1)
        if b.shape[1] in (5, 7, 9):
            raise NotImplementedError("OBB boxes are out of scope for the B200 ReID path")
        if b.shape[1] < 4:
            raise ValueError("Expected detections with at least 4 coordinates")
        return np.ascontiguousarray(b[:, :4])

    # ---- the one-call path ---------------------------------------------------------------------------
    def get_features(self, xyxys, img) -> np.ndarray:
        boxes = self._boxes(xyxys)
        if len(boxes) == 0:
            return np.array([])
        img = np.ascontiguousarray(img, dtype=np.uint8)
        out = np.empty((len(boxes), self.feature_dim), np.float32)
        ok = self.lib.boxmot_reid_capi_compute_features(self.handle, boxes.ctypes.data, len(boxes), img.ctypes.data,
                                                        img.shape[0], img.shape[1], img.shape[2], out.ctypes.data,
                                                        out.size)
        if not ok:
            raise B200Error(self._err())
        return out.astype(np.float16) if self.half else out

    # ---- the staged quartet (utils/timing.py:34-75 drives these) ---------------------------------------
    def get_crops(self, xyxys, img) -> _StagedCrops:
        boxes = self._boxes(xyxys)
        img = np.ascontiguousarray(img, dtype=np.uint8)
        ok = self.lib.boxmot_reid_capi_preprocess(self.handle, boxes.ctypes.data, len(boxes), img.ctypes.data,
                                                  img.shape[0], img.shape[1], img.shape[2])
        if not ok:
            raise B200Error(self._err())
        return _StagedCrops(len(boxes))

    def inference_preprocess(self, crops: _StagedCrops) -> _StagedCrops:
        return crops

    def forward(self, crops: _StagedCrops) -> _StagedCrops:
        if not self.lib.boxmot_reid_capi_process(self.handle):
            raise B200Error(self._err())
        return crops

    def inference_postprocess(self, crops: _StagedCrops) -> np.ndarray:
        out = np.empty((crops.n, self.feature_dim), np.float32)
        if not self.lib.boxmot_reid_capi_postprocess(self.handle, out.ctypes.data, out.size):
            raise B200Error(self._err())
        return out.astype(np.float16) if self.half else out

    def warmup(self, imgsz=None):
        im = np.zeros(imgsz[0] if imgsz else (*self.input_shape, 3), dtype=np.uint8)
        self.get_features(np.array([[0, 0, 64, 64], [0, 0, 128, 128]], np.float32), im)

    # ---- diagnostics --------------------------------------------------------------------------------------
    def debug_stage(self, xyxys, img, stage: int) -> np.ndarray:
        """NHWC float32 activation after `stage` (see include/boxmot_b200.h) for the given boxes."""
        boxes = self._boxes(xyxys)
        img = np.ascontiguousarray(img, dtype=np.uint8)
        per = ctypes.c_int(0)
        # the largest tap: the stem output of the CNNs; CLIP's token maps (at most 257 x 768) are smaller
        cap = len(boxes) * max((self.input_shape[0] // 2) * 64 * 64, 257 * 768)
        out = np.empty(cap, np.float32)
        ok = self.lib.boxmot_b200_reid_debug_stage(self.handle, boxes.ctypes.data, len(boxes), img.ctypes.data,
                                                   img.shape[0], img.shape[1], stage, out.ctypes.data, cap,
                                                   ctypes.byref(per))
        if not ok:
            raise B200Error(_lib.last_error(self.lib))
        return out[: len(boxes) * per.value].reshape(len(boxes), -1).copy()
