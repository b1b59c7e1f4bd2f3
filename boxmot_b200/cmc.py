"""Camera-motion estimators that run on the device.

``SOF`` is a drop-in for the reference's ``boxmot.motion.cmc.sof.SOF`` (and ``get_cmc_method("sof")()``): corners,
cornerSubPix on the initialising frame, pyramidal Lucas-Kanade and a RANSAC partial-affine fit, all as sm_90a CUDA
kernels (boxmot_b200/csrc/cmc_sof.cuh).  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib

SOF_INIT, SOF_ESTIMATED, SOF_REJECTED = 0, 1, 2


class SOF:
    """Sparse-optical-flow camera-motion estimator with the reference's parameters and defaults.

    ``apply(img, dets=None)`` takes a BGR ``uint8`` frame (H, W, 3) and optional detections (N, >=4, xyxy in frame
    pixels; their boxes are left out of the corner search) and returns the float32 (2, 3) warp from the previous frame
    to this one.  The identity comes back on the first frame and when the estimate is rejected; ``last_status`` tells
    which (``SOF_INIT``, ``SOF_ESTIMATED`` or ``SOF_REJECTED``).  A frame of a new size starts the estimator afresh.
    """

    def __init__(self, scale: float = 0.15, min_inliers: int = 8, min_inlier_ratio: float = 0.2,
                 ransac_reproj_threshold: float = 3.0) -> None:
        self.scale = float(scale)
        self.grayscale = True
        self.min_inliers = int(min_inliers)
        self.min_inlier_ratio = float(min_inlier_ratio)
        self.ransac_reproj_threshold = float(ransac_reproj_threshold)
        self.last_status = None
        self._lib = _lib.require_device()
        self._h = self._lib.boxmot_b200_cmc_sof_create(self.scale, self.min_inliers, self.min_inlier_ratio,
                                                       self.ransac_reproj_threshold)
        if not self._h:
            raise _lib.B200Error(f"boxmot_b200_cmc_sof_create: {_lib.last_error(self._lib)}")

    def apply(self, img: np.ndarray, dets: np.ndarray | None = None) -> np.ndarray:
        if img is None or not hasattr(img, "shape") or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError("SOF.apply expects a BGR uint8 frame of shape (H, W, 3)")
        im = np.ascontiguousarray(img, dtype=np.uint8)
        d = np.zeros((0, 4), np.float32)
        if dets is not None:
            a = np.asarray(dets)
            if a.size:
                if a.ndim != 2 or a.shape[1] < 4:
                    raise ValueError("dets must be (N, >=4) xyxy boxes")
                d = np.ascontiguousarray(a[:, :4], dtype=np.float32)
        warp = np.zeros((2, 3), np.float32)
        st = ctypes.c_int(-1)
        ok = self._lib.boxmot_b200_cmc_sof_apply(self._h, im.ctypes.data, im.shape[0], im.shape[1],
                                                 d.ctypes.data if len(d) else None, len(d), warp.ctypes.data,
                                                 ctypes.byref(st))
        if ok != 1:
            raise _lib.B200Error(f"boxmot_b200_cmc_sof_apply: {_lib.last_error(self._lib)}")
        self.last_status = st.value
        return warp

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.boxmot_b200_cmc_sof_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()
