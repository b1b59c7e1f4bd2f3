"""Oracle restatement of BoostTrack / BoostTrack++'s per-frame update -- TEST INFRASTRUCTURE ONLY.

Follows (relative to /root/reference/boxmot):
  * trackers/bbox/boosttrack/boosttrack.py:66-207   KalmanBoxTracker (XYHR filter, confidence, camera_update)
  * trackers/bbox/boosttrack/boosttrack.py:298-529  BoostTrack._update_impl, filter_outputs, the Mahalanobis matrix,
                                                    DLO and DUO confidence boosts
  * trackers/bbox/boosttrack/assoc.py:9-201         shape similarity v1 / v2, Mahalanobis softmax, IoU, soft BIoU,
                                                    match (1-1 shortcut or lapjv(extend_cost=True)), validity filter
  * motion/kalman_filters/xyhr.py:10-102,159-377    8-state [x, y, h, r, vx, vy, vh, vr] filter, constant Q and R
Each track is a plain record (mean, covariance, counters, embedding).  The numpy operations are the reference's, in the
reference's order, so on one machine the oracle and the reference class produce the same bits.  Ids start at 1 per
instance (the reference's class-level counter keeps counting across instances).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from oracle.lap import lapjv

MH_LIMIT = 13.2767            # chi2inv(0.99, 4), the Mahalanobis gate of the boosts and the softmax
_F = np.eye(8)
for _i in range(4):
    _F[_i, 4 + _i] = 1.0
_H = np.eye(4, 8)
_Q = np.eye(8)
_Q[4:, 4:] *= 0.01
_R = np.diag([1.0, 1.0, 10.0, 0.01])


def box_to_z(b):
    w = b[2] - b[0]
    h = b[3] - b[1]
    return np.array([b[0] + w / 2.0, b[1] + h / 2.0, h, w / float(h + 1e-6)])


def x_to_box(x):
    h, r = x[2], x[3]
    w = 0 if r <= 0 else r * h
    return np.array([x[0] - w / 2.0, x[1] - h / 2.0, x[0] + w / 2.0, x[1] + h / 2.0])


def _clamp_geometry(v):
    # python's max(): a NaN stays NaN
    v[2] = max(float(v[2]), 1e-4)
    v[3] = max(float(v[3]), 1e-4)
    return v


class Track:
    """One KalmanBoxTracker as a record."""

    def __init__(self, det, tid, emb):
        self.id, self.conf, self.cls, self.det_ind = tid, det[4], det[5], det[6]
        self.x = np.zeros(8)
        self.x[:4] = _clamp_geometry(box_to_z(det[:4]).copy())
        self.x = _clamp_geometry(self.x)
        self.P = np.diag([10.0] * 4 + [10000.0] * 4)
        self.emb = emb
        self.age = self.hit_streak = self.tsu = 0

    def _enforce(self):
        self.x = _clamp_geometry(self.x)
        self.P = 0.5 * (self.P + self.P.T)

    def predict(self):
        self.x = np.dot(_F, self.x)
        self.P = np.linalg.multi_dot((_F, self.P, _F.T)) + _Q
        self._enforce()
        self.age += 1
        if self.tsu > 0:
            self.hit_streak = 0
        self.tsu += 1

    def confidence(self):
        return 0.9 ** (7 - self.age) if self.age < 7 else 0.9 ** (self.tsu - 1)

    def update(self, det):
        self.tsu = 0
        self.hit_streak += 1
        m = _clamp_geometry(box_to_z(det[:4]).copy())
        S = np.linalg.multi_dot((_H, self.P, _H.T)) + _R
        c, low = scipy.linalg.cho_factor(S, lower=True, check_finite=False)
        K = scipy.linalg.cho_solve((c, low), np.dot(self.P, _H.T).T, check_finite=False).T
        innov = m - np.dot(_H, self.x)
        self.x = self.x + 1.0 * np.dot(innov, K.T)
        self.P = self.P - np.linalg.multi_dot((K, S, K.T))
        self._enforce()
        self.conf, self.cls, self.det_ind = det[4], det[5], det[6]

    def update_emb(self, emb, alpha):
        self.emb = alpha * self.emb + (1 - alpha) * emb
        self.emb /= np.linalg.norm(self.emb)

    def camera_update(self, warp):
        wm = np.vstack([np.asarray(warp, dtype=float).reshape(2, 3), [0.0, 0.0, 1.0]])
        x1, y1, x2, y2 = x_to_box(self.x)
        p1 = wm @ np.array([x1, y1, 1.0])
        p2 = wm @ np.array([x2, y2, 1.0])
        w, h = p2[0] - p1[0], p2[1] - p1[1]
        self.x[:4] = [p1[0] + w / 2, p1[1] + h / 2, h, w / h]


def iou_matrix(a, b):
    a, b = a[:, None, :], b[None, :, :]
    w = np.maximum(0.0, np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]))
    h = np.maximum(0.0, np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]))
    wh = w * h
    return wh / ((a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1]) + (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1]) - wh)


def soft_biou_matrix(d, t):
    """Detections widened by k1 = 0.25, tracks by k2 = 0.5, both times (1 - track confidence)."""
    d, t = d[:, None, :], t[None, :, :]
    s = 1 - t[..., 4]
    dw, dh, tw, th = d[..., 2] - d[..., 0], d[..., 3] - d[..., 1], t[..., 2] - t[..., 0], t[..., 3] - t[..., 1]
    a0, a1, a2, a3 = d[..., 0] - dw * s * 0.25, d[..., 1] - dh * s * 0.25, d[..., 2] + dw * s * 0.25, d[..., 3] + dh * s * 0.25
    b0, b1, b2, b3 = t[..., 0] - tw * s * 0.5, t[..., 1] - th * s * 0.5, t[..., 2] + tw * s * 0.5, t[..., 3] + th * s * 0.5
    w = np.maximum(0.0, np.minimum(a2, b2) - np.maximum(a0, b0))
    h = np.maximum(0.0, np.minimum(a3, b3) - np.maximum(a1, b1))
    wh = w * h
    return wh / ((a2 - a0) * (a3 - a1) + (b2 - b0) * (b3 - b1) - wh)


def shape_matrix(d, t, corrected):
    dw, dh = (d[:, 2] - d[:, 0])[:, None], (d[:, 3] - d[:, 1])[:, None]
    tw, th = (t[:, 2] - t[:, 0])[None, :], (t[:, 3] - t[:, 1])[None, :]
    hden = np.maximum(dh, th) if corrected else np.maximum(dw, tw)
    return np.exp(-(np.abs(dw - tw) / np.maximum(dw, tw) + np.abs(dh - th) / hden))


def mh_matrix(dets, tracks):
    z = np.array([box_to_z(r) for r in dets]).reshape(-1, 4)
    x = np.array([t.x[:4] for t in tracks]).reshape(-1, 4)
    sinv = np.array([np.reciprocal(np.diag(t.P[:4, :4])) for t in tracks]).reshape(-1, 4)
    return ((z[:, None, :] - x[None, :, :]) ** 2 * sinv[None, :, :]).sum(axis=2)


def mh_similarity(md):
    """Gate at MH_LIMIT, then a softmax of (limit - distance) over the detections of each track column."""
    mask = md > MH_LIMIT
    v = MH_LIMIT - np.where(mask, MH_LIMIT, md)
    return np.where(mask, 0, np.exp(v) / np.exp(v).sum(0).reshape((1, -1)))


def match(cost, threshold):
    if cost.size == 0:
        return np.empty((0, 2), dtype=int)
    a = (cost > threshold).astype(np.int32)
    if a.sum(1).max() == 1 and a.sum(0).max() == 1:
        return np.stack(np.where(a), axis=1)
    _, x, _ = lapjv(-cost, extend_cost=True)
    return np.array([[r, c] for r, c in enumerate(x) if c >= 0], dtype=int).reshape(-1, 2)


class BoostTrackOracle:
    def __init__(self, reid_model=None, min_box_area=10, aspect_ratio_thresh=1.6, lambda_iou=0.5, lambda_mhd=0.25,
                 lambda_shape=0.25, use_dlo_boost=True, use_duo_boost=True, dlo_boost_coef=0.65, s_sim_corr=False,
                 use_rich_s=False, use_sb=False, use_vt=False, with_reid=False, det_thresh=0.3, max_age=30, min_hits=3,
                 iou_threshold=0.3):
        self.min_box_area, self.ar_thresh = min_box_area, aspect_ratio_thresh
        self.l_iou, self.l_mhd, self.l_shape = lambda_iou, lambda_mhd, lambda_shape
        self.dlo, self.duo, self.dlo_coef, self.s_corr = use_dlo_boost, use_duo_boost, dlo_boost_coef, s_sim_corr
        self.rich_s, self.sb, self.vt = use_rich_s, use_sb, use_vt
        self.with_reid = bool(with_reid) and reid_model is not None
        self.model = reid_model
        self.det_thresh, self.max_age, self.min_hits, self.iou_threshold = det_thresh, max_age, min_hits, iou_threshold
        self.tracks: list[Track] = []
        self.frame_count = 0
        self._next = 1

    # ---- confidence boosts ----
    def _dlo(self, d):
        if len(d) == 0 or not self.tracks:
            return d
        boxes = np.array([np.r_[x_to_box(t.x), t.confidence()] for t in self.tracks])
        if self.rich_s:
            S = (mh_similarity(mh_matrix(d, self.tracks)) + shape_matrix(d, boxes, self.s_corr)
                 + soft_biou_matrix(d, boxes)) / 3
        else:
            S = iou_matrix(d, boxes)
        if not self.sb and not self.vt:
            d[:, 4] = np.maximum(d[:, 4], S.max(1) * self.dlo_coef)
            return d
        if self.sb:
            d[:, 4] = np.maximum(d[:, 4], 0.65 * d[:, 4] + (1 - 0.65) * S.max(1) ** 1.5)
        if self.vt:
            lim = np.maximum(0.95 - np.array([t.tsu - 1 for t in self.tracks]), 0.8)
            hit = (S > lim).max(1)
            sc = d[:, 4].copy()
            sc[hit] = np.maximum(sc[hit], self.det_thresh + 1e-5)
            d[:, 4] = sc
        return d

    def _duo(self, d):
        if len(d) == 0 or not self.tracks:
            return d
        cand = np.where((mh_matrix(d, self.tracks).min(1) > MH_LIMIT) & (d[:, 4] < self.det_thresh))[0]
        if len(cand) == 0:
            return d
        ov = iou_matrix(d[cand], d[cand]) - np.eye(len(cand))
        ovmax = ov.max(axis=1)
        keep = list(cand[ovmax <= 0.3])
        crowded = np.where(ovmax > 0.3)[0]
        for i in crowded:
            group = np.append(np.intersect1d(cand[crowded], cand[ov[i] > 0.3]), cand[i])
            if d[cand[i], 4] == np.max(d[group, 4]):
                keep.append(cand[i])
        d[np.asarray(keep, dtype=int), 4] = self.det_thresh + 1e-4
        return d

    def update(self, dets, img=None, embs=None, warp=None):
        """`warp`: the 2x3 matrix the reference's camera-motion estimator returns for this frame (applied to every
        track before the predict step); None = no camera-motion compensation."""
        dets = np.asarray(dets)
        if dets.size == 0:
            dets = np.empty((0, 6), dtype=np.float32)
        assert dets.ndim == 2 and dets.shape[1] == 6
        d = np.hstack([dets, np.arange(len(dets)).reshape(-1, 1)])
        self.frame_count += 1
        if warp is not None:
            for t in self.tracks:
                t.camera_update(warp)
        confs = []
        for t in self.tracks:
            t.predict()
            confs.append(t.confidence())
        trks = np.array([np.r_[x_to_box(t.x), c] for t, c in zip(self.tracks, confs)]).reshape(-1, 5)
        if self.dlo:
            d = self._dlo(d)
        if self.duo:
            d = self._duo(d)
        keep = d[:, 4] >= self.det_thresh
        d = d[keep]
        dembs = np.ones((len(d), 1))
        if self.with_reid and len(d):
            dembs = np.asarray(embs)[keep] if embs is not None else self.model.get_features(d[:, :4], img)
        emb_cost = None
        if self.with_reid and self.tracks:
            te = np.array([t.emb for t in self.tracks])
            emb_cost = np.empty((0, len(te))) if len(dembs) == 0 else dembs.reshape(len(dembs), -1) @ te.reshape(len(te), -1).T

        # ---- association ----
        T = len(self.tracks)
        if T == 0:
            matches, und, unt = np.empty((0, 2), dtype=int), list(range(len(d))), []
        else:
            iou = iou_matrix(d, trks)
            cost = iou.copy()
            conf = np.multiply(d[:, 4].reshape(-1, 1), np.array(confs).reshape(1, -1))
            conf[iou < self.iou_threshold] = 0
            cost += self.l_iou * conf * iou_matrix(d, trks)
            if len(d):
                cost += self.l_mhd * mh_similarity(mh_matrix(d, self.tracks))
                cost += self.l_shape * conf * shape_matrix(d, trks, self.s_corr)
            if emb_cost is not None:
                cost += (1 + self.l_iou + self.l_shape + self.l_mhd) * 1.5 * emb_cost
            pairs = match(cost, self.iou_threshold)
            und = [i for i in range(len(d)) if i not in pairs[:, 0]]
            unt = [k for k in range(T) if k not in pairs[:, 1]]
            good = []
            for r, c in pairs:
                ok = iou[r, c] >= self.iou_threshold or (
                    emb_cost is not None and iou[r, c] >= self.iou_threshold / 2 and emb_cost[r, c] >= 0.75)
                if ok:
                    good.append((r, c))
                else:
                    und.append(r)
                    unt.append(c)
            matches = np.array(good, dtype=int).reshape(-1, 2)
        alpha = 0.95 + (1 - 0.95) * (1 - (d[:, 4] - self.det_thresh) / (1 - self.det_thresh))
        for r, c in matches:
            self.tracks[c].update(d[r, :])
            self.tracks[c].update_emb(dembs[r], alpha[r])
        for i in und:
            self.tracks.append(Track(d[i, :], self._next, dembs[i]))
            self._next += 1

        out = []
        for t in self.tracks:
            if t.tsu < 1 and (t.hit_streak >= self.min_hits or self.frame_count <= self.min_hits):
                out.append(np.r_[x_to_box(t.x), t.id, t.conf, t.cls, t.det_ind])
        self.tracks = [t for t in self.tracks if t.tsu <= self.max_age]
        if not out:
            return np.empty((0, 8))
        out = np.vstack(out)
        w, h = out[:, 2] - out[:, 0], out[:, 3] - out[:, 1]
        with np.errstate(divide="ignore", invalid="ignore"):
            return out[(w / h <= self.ar_thresh) & (w * h > self.min_box_area)]

    def state_snapshot(self):
        return {t.id: (t.x.copy(), t.P.copy()) for t in self.tracks}
