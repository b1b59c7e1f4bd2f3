"""Oracle restatement of OccluBoost's per-frame update -- TEST INFRASTRUCTURE ONLY.

Follows (paths in the reference boxmot package), AABB path only:
  * trackers/bbox/occluboost/occluboost.py:185-483  _update_impl: BoostTrack's predict, boosts and association (from
                                                    BoostTrackOracle), then abnormal-motion updates, the ReID recovery
                                                    pass, the low-confidence second pass, online GTA, tentative births,
                                                    duplicate suppression, emit and cull with burial
  * trackers/bbox/occluboost/occluboost.py:485-906  _maybe_activate, the GTA helpers, flush_gta with its Gaussian-process
                                                    smoothing, _compute_ams_alpha, _ams_update,
                                                    _suppress_duplicate_emissions
Tracks are plain records; the numpy, scipy and sklearn calls are the reference's, in the reference's order.  `counts`
records how often each branch fired, so the golden cases can be checked to reach all of them.  Ids start at 1 per
instance.
"""
from __future__ import annotations

from collections import Counter, deque

import numpy as np
import scipy.linalg
from scipy.optimize import linear_sum_assignment

from tests.boosttrack_oracle import MH_LIMIT, BoostTrackOracle, Track, _H, _R, _clamp_geometry, box_to_z, \
    iou_matrix, match, mh_matrix, mh_similarity, shape_matrix, x_to_box  # noqa: F401

OB_DEFAULTS = dict(recovery_appearance_thresh=0.99, recovery_iou_thresh=0.1, recovery_max_age=1, feat_alpha=0.95,
                   track_low_thresh=0.1, second_iou_thresh=0.6, second_appearance_thresh=0.5, second_pass_max_age=1,
                   second_pass_min_hits=3, use_second_pass=False, new_track_thresh=0.6, confirm_hits=2,
                   instant_confirm_thresh=0.7, tentative_max_age=1, duplicate_iou_thresh=0.85, ams_enabled=True,
                   ams_alpha0=0.4, ams_threshold=0.5, ams_buffer_size=30, ams_shrink_ratio=0.75,
                   lambda_emb_multiplier=1.5, gta_enabled=True, gta_appearance_thresh=0.5, gta_min_track_length=5,
                   gta_smooth_tau=5.0, gta_interpolate=True, gta_max_gap=60)


class ObTrack(Track):
    def __init__(self, det, tid, emb, activated):
        super().__init__(det, tid, emb)
        self.activated = activated
        self.buf = None

    def update(self, det, alpha=1.0):
        self.tsu = 0
        self.hit_streak += 1
        m = _clamp_geometry(box_to_z(det[:4]).copy())
        S = np.linalg.multi_dot((_H, self.P, _H.T)) + _R
        c, low = scipy.linalg.cho_factor(S, lower=True, check_finite=False)
        K = scipy.linalg.cho_solve((c, low), np.dot(self.P, _H.T).T, check_finite=False).T
        innov = m - np.dot(_H, self.x)
        self.x = self.x + alpha * np.dot(innov, K.T)
        self.P = self.P - np.linalg.multi_dot((K, S, K.T))
        self._enforce()
        self.conf, self.cls, self.det_ind = det[4], det[5], det[6]


class OccluBoostOracle(BoostTrackOracle):
    def __init__(self, reid_model=None, **kw):
        o = dict(OB_DEFAULTS)
        o.update({k: kw.pop(k) for k in list(kw) if k in OB_DEFAULTS})
        super().__init__(reid_model=reid_model, **kw)
        self.o = o
        self.new_track_thresh = max(o["new_track_thresh"], 0.0)
        self.confirm_hits = max(int(o["confirm_hits"]), 1)
        self.tentative_max_age = max(int(o["tentative_max_age"]), 0)
        self.ams_alpha0 = float(np.clip(o["ams_alpha0"], 0.0, 1.0))
        self.ams_threshold = float(max(o["ams_threshold"], 0.0))
        self.ams_buffer_size = int(max(o["ams_buffer_size"], 2))
        self.ams_shrink_ratio = float(np.clip(o["ams_shrink_ratio"], 0.0, 1.0))
        self.gta = bool(o["gta_enabled"]) and self.with_reid
        self.gta_min_len = max(int(o["gta_min_track_length"]), 1)
        self.gta_max_gap = max(int(o["gta_max_gap"]), 1)
        self.graveyard: dict = {}
        self.gap_rows: list = []
        self.counts = Counter()

    # ---- AMS (occluboost.py:778-865) ----
    def _ams_alpha(self, t, box):
        if not self.o["ams_enabled"] or self.ams_alpha0 >= 1.0:
            return 1.0
        x1, y1, x2, y2 = float(box[0]), float(box[1]), float(box[2]), float(box[3])
        w, h = max(x2 - x1, 1e-6), max(y2 - y1, 1e-6)
        cur = np.array([x1 + 0.5 * w, y1 + 0.5 * h, w, h], dtype=float)
        if t.buf is None:
            t.buf = deque(maxlen=self.ams_buffer_size)
        if len(t.buf) < 2:
            t.buf.append(cur)
            return 1.0
        cur_v = cur - t.buf[-1]
        mean_v = np.diff(np.asarray(t.buf, dtype=float), axis=0).mean(axis=0)
        cur_c, mean_c = float(np.linalg.norm(cur_v[:2])), float(np.linalg.norm(mean_v[:2]))
        cur_a, mean_a = float(np.linalg.norm(cur_v[2:])), float(np.linalg.norm(mean_v[2:]))
        d_c = max(0.0, cur_c - mean_c) / max(mean_c, 1e-6)
        d_a = max(0.0, cur_a - mean_a) / max(mean_a, 1e-6)
        alpha = 0.5 * ((1.0 if d_c <= self.ams_threshold else self.ams_alpha0)
                       + (1.0 if d_a <= self.ams_threshold else self.ams_alpha0))
        mean_area = float(np.mean(np.asarray(t.buf, dtype=float)[:, 2:].prod(axis=1)))
        if float(cur[2] * cur[3]) >= mean_area * self.ams_shrink_ratio:
            alpha = 1.0
        t.buf.append(cur)
        return float(alpha)

    def _ams_update(self, t, det):
        alpha = self._ams_alpha(t, det[:4])
        if alpha < 1.0:
            self.counts["ams_damped"] += 1
        if t.upd_frame == self.frame_count:
            self.counts["updated_twice"] += 1
        t.upd_frame = self.frame_count
        t.update(det, alpha)

    def _activate(self, t):
        if not t.activated and t.hit_streak >= self.confirm_hits:
            t.activated = True

    def _new(self, det, tid, emb, activated):
        t = ObTrack(det, tid, emb, activated)
        t.upd_frame = -1
        return t

    def update(self, dets, img=None, embs=None, warp=None):
        o = self.o
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
        orig = d[:, 4].copy()
        if self.dlo:
            d = self._dlo(d)
        if self.duo:
            d = self._duo(d)
        keep = d[:, 4] >= self.det_thresh
        second = (~keep) & (orig >= o["track_low_thresh"]) & (orig < self.det_thresh) if o["use_second_pass"] \
            else np.zeros_like(keep)
        d_sec = d[second]
        d = d[keep]
        dembs = np.ones((len(d), 1))
        dembs_sec = np.ones((len(d_sec), 1))
        if self.with_reid:
            # the reference embeds the kept and the second-pass rows in two calls; per-row embeddings are the same
            all_e = np.asarray(embs) if embs is not None else np.asarray(self.model.get_features(dets[:, :4], img))
            dembs, dembs_sec = all_e[keep], all_e[second]
        emb_cost = None
        if self.with_reid and self.tracks and len(d):
            te = np.array([t.emb for t in self.tracks])
            emb_cost = dembs.reshape(len(dembs), -1) @ te.reshape(len(te), -1).T

        # ---- association (assoc.py associate with lambda_emb_multiplier) ----
        T = len(self.tracks)
        if T == 0 or len(d) == 0:
            matches, und, unt = np.empty((0, 2), dtype=int), list(range(len(d))), list(range(T))
        else:
            iou = iou_matrix(d, trks)
            cost = iou.copy()
            conf = np.multiply(d[:, 4].reshape(-1, 1), np.array(confs).reshape(1, -1))
            conf[iou < self.iou_threshold] = 0
            cost += self.l_iou * conf * iou_matrix(d, trks)
            cost += self.l_mhd * mh_similarity(mh_matrix(d, self.tracks))
            cost += self.l_shape * conf * shape_matrix(d, trks, self.s_corr)
            if emb_cost is not None:
                cost += (1 + self.l_iou + self.l_shape + self.l_mhd) * o["lambda_emb_multiplier"] * emb_cost
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
            t = self.tracks[c]
            self._ams_update(t, d[r, :])
            if self.with_reid:
                t.update_emb(dembs[r], alpha[r])
            self._activate(t)

        def pos(t):
            return np.r_[x_to_box(t.x), t.confidence()]

        # ---- ReID recovery pass ----
        if self.with_reid and unt and und:
            elig = [k for k in unt if self.tracks[k].tsu <= o["recovery_max_age"]]
            if elig:
                sim = dembs[und].reshape(len(und), -1) @ np.stack([self.tracks[k].emb for k in elig]).reshape(len(elig), -1).T
                ious = iou_matrix(d[und], np.array([pos(self.tracks[k]) for k in elig]))
                g = sim.copy()
                g[ious < o["recovery_iou_thresh"]] = -1.0
                g[sim < o["recovery_appearance_thresh"]] = -1.0
                if (g > 0).any():
                    done = set()
                    for r, c in zip(*linear_sum_assignment(-g)):
                        if g[r, c] <= 0:
                            continue
                        self.counts["recovery"] += 1
                        t = self.tracks[elig[c]]
                        done.add(und[r])
                        self._ams_update(t, d[und[r], :])
                        t.update_emb(dembs[und[r]], alpha=o["feat_alpha"])
                        self._activate(t)
                    und = [i for i in und if i not in done]

        # ---- low-confidence second pass ----
        if o["use_second_pass"] and unt and len(d_sec):
            elig = [k for k in unt if self.tracks[k].tsu <= o["second_pass_max_age"]
                    and self.tracks[k].hit_streak >= o["second_pass_min_hits"] and self.tracks[k].activated]
            if elig:
                ious2 = iou_matrix(d_sec, np.array([pos(self.tracks[k]) for k in elig]))
                cost = 1.0 - ious2
                cost[ious2 < o["second_iou_thresh"]] = 1.0
                if self.with_reid and len(dembs_sec):
                    sim2 = dembs_sec.reshape(len(dembs_sec), -1) @ np.stack([self.tracks[k].emb for k in elig]).reshape(len(elig), -1).T
                    cost[sim2 < o["second_appearance_thresh"]] = 1.0
                if (cost < 1.0).any():
                    used = set()
                    for r, c in zip(*linear_sum_assignment(cost)):
                        if cost[r, c] >= 1.0 or elig[c] in used:
                            continue
                        used.add(elig[c])
                        self.counts["second"] += 1
                        t = self.tracks[elig[c]]
                        self._ams_update(t, d_sec[r, :])
                        if self.with_reid and len(dembs_sec):
                            t.update_emb(dembs_sec[r], alpha=o["feat_alpha"])
                        self._activate(t)

        # ---- GTA appearance recovery ----
        if self.gta and und and unt:
            elig = [k for k in unt if self.tracks[k].tsu <= self.gta_max_gap and self.tracks[k].age >= self.gta_min_len]
            if elig:
                sim = dembs[und].reshape(len(und), -1) @ np.stack([self.tracks[k].emb for k in elig]).reshape(len(elig), -1).T
                g = sim.copy()
                g[sim < o["gta_appearance_thresh"]] = -1.0
                if (g > 0).any():
                    done = set()
                    for r, c in zip(*linear_sum_assignment(-g)):
                        if g[r, c] <= 0:
                            continue
                        self.counts["gta_recovery"] += 1
                        t = self.tracks[elig[c]]
                        done.add(und[r])
                        self._ams_update(t, d[und[r], :])
                        t.update_emb(dembs[und[r]], alpha=o["feat_alpha"])
                        self._activate(t)
                    und = [i for i in und if i not in done]

        # ---- GTA resurrection ----
        if self.gta and und and self.graveyard:
            gids = list(self.graveyard)
            sim = dembs[und].reshape(len(und), -1) @ np.stack([self.graveyard[k]["emb"] for k in gids]).reshape(len(gids), -1).T
            g = sim.copy()
            g[sim < o["gta_appearance_thresh"]] = -1.0
            if (g > 0).any():
                done = set()
                for r, c in zip(*linear_sum_assignment(-g)):
                    if g[r, c] <= 0:
                        continue
                    i, gid = und[r], gids[c]
                    entry = self.graveyard[gid]
                    if d[i, 4] < self.new_track_thresh:
                        self.counts["resurrect_low_conf"] += 1
                        continue
                    done.add(i)
                    t = self._new(d[i, :], gid, dembs[i] if self.with_reid else None, True)
                    self.tracks.append(t)
                    self.counts["resurrect"] += 1
                    if o["gta_interpolate"]:
                        gap = self.frame_count - entry["frame"]
                        if 1 < gap <= self.gta_max_gap:
                            self.counts["gap_rows"] += gap - 1
                            last, cur = entry["last_box"], x_to_box(t.x)
                            for k in range(1, gap):
                                a = k / gap
                                b = (1.0 - a) * last + a * cur
                                self.gap_rows.append(np.array([entry["frame"] + k, gid, b[0], b[1], b[2], b[3],
                                                               entry["conf"], entry["cls"], -1.0], dtype=float))
                    del self.graveyard[gid]
                und = [i for i in und if i not in done]

        for i in und:
            if d[i, 4] >= self.new_track_thresh:
                act = bool(d[i, 4] >= o["instant_confirm_thresh"] or self.confirm_hits <= 1)
                self.tracks.append(self._new(d[i, :], self._next, dembs[i] if self.with_reid else None, act))
                self._next += 1

        emitted = [t for t in self.tracks if t.tsu < 1 and t.activated
                   and (t.hit_streak >= self.min_hits or self.frame_count <= self.min_hits)]
        if len(emitted) > 1 and 0.0 < o["duplicate_iou_thresh"] < 1.0:
            boxes = np.stack([x_to_box(t.x) for t in emitted])
            ious = iou_matrix(boxes, boxes)
            np.fill_diagonal(ious, 0.0)
            drop = set()
            for i in range(len(emitted)):
                if i in drop:
                    continue
                for j in range(i + 1, len(emitted)):
                    if j in drop:
                        continue
                    if ious[i, j] >= o["duplicate_iou_thresh"]:
                        drop.add(j if emitted[i].age >= emitted[j].age else i)
            if drop:
                self.counts["duplicate_drop"] += len(drop)
                ids = {emitted[k].id for k in drop}
                self.tracks = [t for t in self.tracks if t.id not in ids]
                emitted = [t for k, t in enumerate(emitted) if k not in drop]
        out = [np.r_[x_to_box(t.x), t.id, t.conf, t.cls, t.det_ind] for t in emitted]

        alive = []
        for t in self.tracks:
            if t.tsu <= self.max_age and (t.activated or t.tsu <= self.tentative_max_age):
                alive.append(t)
                continue
            if not t.activated and t.tsu <= self.max_age:
                self.counts["tentative_expired"] += 1
            if self.gta and t.age >= self.gta_min_len:
                self.counts["buried"] += 1
                self.graveyard[t.id] = dict(emb=t.emb.copy(), last_box=x_to_box(t.x).copy(), frame=self.frame_count,
                                            conf=float(t.conf), cls=float(t.cls))
        for gid in [k for k, v in self.graveyard.items() if self.frame_count - v["frame"] > self.gta_max_gap]:
            del self.graveyard[gid]
        self.tracks = alive
        if not out:
            return np.empty((0, 8))
        out = np.vstack(out)
        w, h = out[:, 2] - out[:, 0], out[:, 3] - out[:, 1]
        with np.errstate(divide="ignore", invalid="ignore"):
            return out[(w / h <= self.ar_thresh) & (w * h > self.min_box_area)]

    def flush_gta(self):
        if not self.gap_rows:
            return np.empty((0, 9))
        rows = list(self.gap_rows)
        tau = self.o["gta_smooth_tau"]
        if tau > 0 and len(rows) >= 3:
            from sklearn.gaussian_process import GaussianProcessRegressor
            from sklearn.gaussian_process.kernels import RBF

            groups: dict = {}
            for k, r in enumerate(rows):
                groups.setdefault(int(r[1]), []).append(k)
            for idx in groups.values():
                if len(idx) < 3:
                    continue
                frames = np.array([rows[k][0] for k in idx]).reshape(-1, 1)
                boxes = np.array([rows[k][2:6] for k in idx])
                ls = np.clip(tau * np.log(max(tau ** 3 / len(idx), 1e-6)), tau ** -1, tau ** 2)
                sm = GaussianProcessRegressor(RBF(ls, length_scale_bounds="fixed")).fit(frames, boxes).predict(frames)
                for j, k in enumerate(idx):
                    rows[k][2:6] = sm[j]
        self.gap_rows = []
        self.graveyard = {}
        return np.vstack(rows)

    def state_snapshot(self):
        return {t.id: (t.x.copy(), t.P.copy(), t.activated) for t in self.tracks}
