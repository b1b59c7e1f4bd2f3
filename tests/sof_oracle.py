"""SofOracle: `SOF.apply` of the reference (boxmot/motion/cmc/sof.py with base_cmc.py) restated on the installed OpenCV.

Test infrastructure only, like the ECC reference in tests/test_zzgpu_cmc.py: the same cv2 calls with the same
parameters and the same decisions, without the reference package (which is not present where the GPU tests run).
`status` after apply: 0 initialising frame, 1 estimated, 2 rejected.
"""
from __future__ import annotations

import numpy as np

import cv2

CORNERS = dict(maxCorners=1000, qualityLevel=0.01, minDistance=1, blockSize=3, useHarrisDetector=False, k=0.04)
LK = dict(winSize=(21, 21), maxLevel=3, criteria=(cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 30, 0.01))
SUBPIX_CRIT = (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 30, 0.01)


def preprocess(img, scale=0.15):
    return cv2.resize(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), (0, 0), fx=scale, fy=scale, interpolation=cv2.INTER_LINEAR)


def corner_mask(gray, dets, scale=0.15):
    """Keep the central 2 %..98 % band, clear every detection box (float32 coordinates * scale, truncated)."""
    h, w = gray.shape
    m = np.zeros((h, w), np.uint8)
    m[int(0.02 * h):int(0.98 * h), int(0.02 * w):int(0.98 * w)] = 255
    for d in ([] if dets is None else np.asarray(dets)):
        if len(d) < 4:
            continue
        x1, y1, x2, y2 = (np.asarray(d[:4], dtype=np.float32) * np.float32(scale)).astype(int).tolist()
        x1, x2 = max(0, min(w, x1)), max(0, min(w, x2))
        y1, y2 = max(0, min(h, y1)), max(0, min(h, y2))
        if x2 > x1 and y2 > y1:
            m[y1:y2, x1:x2] = 0
    return m


class SofOracle:
    def __init__(self, scale=0.15, min_inliers=8, min_inlier_ratio=0.2, ransac_reproj_threshold=3.0):
        self.scale, self.min_inliers, self.min_ratio = scale, min_inliers, min_inlier_ratio
        self.thr = ransac_reproj_threshold
        self.prev, self.kps, self.ready = None, None, False
        self.status, self.n_valid, self.n_inliers = None, 0, 0

    def _corners(self, gray, dets):
        return cv2.goodFeaturesToTrack(gray, mask=corner_mask(gray, dets, self.scale), **CORNERS)

    def apply(self, img, dets=None):
        gray = preprocess(img, self.scale)
        eye = np.eye(2, 3, dtype=np.float32)
        if not self.ready:
            kps = self._corners(gray, dets)
            self.status, self.prev = 0, gray
            if kps is None or len(kps) < 4:
                self.kps, self.ready = kps, False
                return eye
            cv2.cornerSubPix(gray, kps, (5, 5), (-1, -1), SUBPIX_CRIT)
            self.kps, self.ready = kps, True
            return eye
        nxt, st, _ = cv2.calcOpticalFlowPyrLK(self.prev, gray, self.kps, None, **LK)
        st = st.reshape(-1) == 1
        pv, nv = self.kps[st], nxt[st]
        self.n_valid, self.n_inliers, self.status = len(pv), 0, 2
        if len(pv) < 4:
            kps = self._corners(gray, dets)
            self.prev, self.kps = gray, kps
            self.ready = kps is not None and len(kps) >= 4
            return eye
        H, inl = cv2.estimateAffinePartial2D(pv, nv, method=cv2.RANSAC, ransacReprojThreshold=self.thr)
        out = eye
        if H is not None:
            self.n_inliers = int(np.count_nonzero(inl))
            if self.n_inliers >= self.min_inliers and self.n_inliers / len(pv) >= self.min_ratio:
                out = H.astype(np.float32)
                if self.scale < 1.0:
                    out[0, 2] /= self.scale
                    out[1, 2] /= self.scale
                self.status = 1
        kps = self._corners(gray, dets)
        self.prev, self.kps, self.ready = gray, (nv if kps is None or len(kps) < 4 else kps), True
        return out
