"""Plain-record restatement of SFSORT (boxmot/trackers/bbox/sfsort/sfsort.py, AABB path) -- TEST INFRASTRUCTURE ONLY.

The device core (boxmot_b200/csrc/sf_core.cuh) is checked against this oracle and this oracle against the reference's
goldens.  Comparison precision is explicit here instead of following numpy's weak-scalar rules: a threshold compares in
float64 when the reference holds it as np.float64 (the density-tuned thresholds), in float32 otherwise.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle.lap import lapjv

ACTIVE, LOST_CENTRAL, LOST_MARGINAL = 0, 1, 2
F32 = np.float32
EPS = F32(1e-7)


def _clamp(v, lo, hi):
    return max(lo, min(v, hi))


def resolve(high_th=0.6, match_th_first=0.67, new_track_th=0.7, low_th=0.1, match_th_second=0.3, dynamic_tuning=False,
            cth=0.5, high_th_m=0.0, new_track_th_m=0.0, match_th_first_m=0.0, marginal_timeout=0, central_timeout=0,
            frame_width=None, frame_height=None, horizontal_margin=None, vertical_margin=None, **_ignored):
    """The constructor's `_resolve_or_default` clamps (sfsort.py:205-237)."""
    def rd(v, d, lo, hi):
        return _clamp(d if v is None else v, lo, hi)

    r = dict(high_th=float(rd(high_th, 0.6, 0.0, 1.0)))
    r["match_th_first"] = float(rd(match_th_first, 0.67, 0.0, 0.67))
    r["new_track_th"] = float(rd(new_track_th, 0.7, r["high_th"], 1.0))
    r["low_th"] = float(rd(low_th, 0.1, 0.0, r["high_th"]))
    r["match_th_second"] = float(rd(match_th_second, 0.3, 0.0, 1.0))
    r["dynamic_tuning"] = bool(dynamic_tuning)
    r["cth"] = float(rd(cth, 0.5, r["low_th"], 1.0))
    if dynamic_tuning:
        r["high_th_m"] = float(rd(high_th_m, 0.0, 0.02, 0.1))
        r["new_track_th_m"] = float(rd(new_track_th_m, 0.0, 0.02, 0.08))
        r["match_th_first_m"] = float(rd(match_th_first_m, 0.0, 0.02, 0.08))
    else:
        r["high_th_m"] = 0.0 if high_th_m is None else float(high_th_m)
        r["new_track_th_m"] = 0.0 if new_track_th_m is None else float(new_track_th_m)
        r["match_th_first_m"] = 0.0 if match_th_first_m is None else float(match_th_first_m)
    r["marginal_timeout"] = int(rd(marginal_timeout, 0, 0, 500))
    r["central_timeout"] = int(rd(central_timeout, 0, 0, 1000))
    r["frame_width"], r["frame_height"] = frame_width, frame_height
    r["horizontal_margin"] = horizontal_margin or 0
    r["vertical_margin"] = vertical_margin or 0
    return r


def margins(w, h, hm, vm):
    """(l, r, t, b) of `_maybe_set_margins`; a margin of 0 is the same as None."""
    return (float(_clamp(hm, 0, w)), float(_clamp(w - hm, 0, w)), float(_clamp(vm, 0, h)), float(_clamp(h - vm, 0, h)))


def gt(score, th, f64):
    """score (float32) > th, compared in float64 or in float32."""
    return float(score) > th if f64 else F32(score) > F32(th)


def cost_matrix(tb, db, iou_only):
    """`_calculate_cost_aabb` + `_combine_cost_terms` in float32, numpy's order of operations."""
    tb = np.asarray(tb, F32).reshape(-1, 4)
    db = np.asarray(db, F32).reshape(-1, 4)
    with np.errstate(all="ignore"):
        a0, a1, a2, a3 = (tb[:, k][:, None] for k in range(4))
        b0, b1, b2, b3 = (db[:, k][None, :] for k in range(4))
        hi = np.maximum(np.minimum(a2, b2) - np.maximum(a0, b0), F32(0))
        wi = np.maximum(np.minimum(a3, b3) - np.maximum(a1, b1), F32(0))
        inter = hi * wi
        bh1, bh2, bw1, bw2 = a2 - a0, b2 - b0, a3 - a1, b3 - b1
        union = ((bh2 * bw2 + bh1 * bw1) - inter) + EPS
        iou = inter / union
        if iou_only:
            return F32(1) - iou
        cx1, cy1, cx2, cy2 = (a0 + a2) / F32(2), (a1 + a3) / F32(2), (b0 + b2) / F32(2), (b1 + b3) / F32(2)
        sw = wi / np.abs((wi + np.abs(bw2 - bw1)) + EPS)
        sh = hi / np.abs((hi + np.abs(bh2 - bh1)) + EPS)
        inner = np.abs(cx1 - cx2) + np.abs(cy1 - cy2)
        outer = np.abs(np.maximum(a2, b2) - np.minimum(a0, b0)) + np.abs(np.maximum(a3, b3) - np.minimum(a1, b1))
        outer = np.maximum(outer, EPS)
        diou = iou - inner / outer
        return F32(1) - ((diou + sh) + sw) / F32(3)


@dataclass(eq=False)
class Track:
    box: np.ndarray
    last_frame: int
    id: int
    conf: np.float32
    cls: np.float32
    det_ind: int
    state: int = ACTIVE


@dataclass
class SfOracle:
    cfg: dict
    active: list = field(default_factory=list)
    lost: list = field(default_factory=list)
    frame: int = 0
    next_id: int = 0
    mrg: tuple = None
    hits: dict = field(default_factory=dict)

    def __post_init__(self):
        c = self.cfg
        if c["frame_width"] is not None and c["frame_height"] is not None:
            self.mrg = margins(c["frame_width"], c["frame_height"], c["horizontal_margin"], c["vertical_margin"])

    def _hit(self, k):
        self.hits[k] = self.hits.get(k, 0) + 1

    def _thresholds(self, scores):
        c = self.cfg
        hth, nth, mth = c["high_th"], c["new_track_th"], c["match_th_first"]
        if not c["dynamic_tuning"]:
            return hth, nth, mth, False
        count = max(int(np.sum(scores > F32(c["cth"]))), 1)
        lnc = float(np.log10(count))
        hth = _clamp(hth - c["high_th_m"] * lnc, 0.0, 1.0)
        nth = _clamp(nth + c["new_track_th_m"] * lnc, hth, 1.0)
        mth = _clamp(mth - c["match_th_first_m"] * lnc, 0.0, 0.67)
        return hth, nth, mth, True

    def _birth(self, d, row):
        t = Track(d[:4].copy(), self.frame, self.next_id, d[4], d[5], row)
        self.next_id += 1
        self._hit("birth")
        return t

    @staticmethod
    def _update(t, d, frame, row):
        t.box, t.last_frame, t.conf, t.cls, t.det_ind, t.state = d[:4].copy(), frame, d[4], d[5], row, ACTIVE

    def update(self, dets, hw=None):
        dets = np.asarray(dets, F32).reshape(-1, 6)
        c = self.cfg
        if self.mrg is None and hw is not None:
            self.mrg = margins(hw[1], hw[0], c["horizontal_margin"], c["vertical_margin"])
        self.frame += 1
        scores = dets[:, 4]
        hth, nth, mth, f64 = self._thresholds(scores)
        for t in list(self.lost):   # purge
            timeout = c["central_timeout"] if t.state == LOST_CENTRAL else c["marginal_timeout"]
            if self.frame - t.last_frame > timeout:
                self.lost.remove(t)
                self._hit("purge_central" if t.state == LOST_CENTRAL else "purge_marginal")
        pool = self.active + self.lost
        nxt = []
        high = [i for i in range(len(dets)) if gt(scores[i], hth, f64)]
        mid = [i for i in range(len(dets))
               if F32(c["low_th"]) < scores[i] and (float(scores[i]) < hth if f64 else scores[i] < F32(hth))]
        if any(float(s) == hth for s in scores) or (not f64 and any(F32(s) == F32(hth) for s in scores)):
            self._hit("score_at_hth")
        unmatched = None   # the reference's `unmatched_tracks`: None while it is the initial empty array
        if high:
            if pool:
                cost = cost_matrix([t.box for t in pool], dets[high, :4], False).astype(np.float64)
                _, x, y = lapjv(cost, extend_cost=True, cost_limit=mth)
                for r in range(len(pool)):
                    if x[r] >= 0:
                        t = pool[r]
                        self._update(t, dets[high[x[r]]], self.frame, high[x[r]])
                        nxt.append(t)
                        if t in self.lost:
                            self.lost.remove(t)
                            self._hit("reacquire_pass1")
                for k in range(len(high)):
                    if y[k] < 0 and gt(scores[high[k]], nth, f64):
                        nxt.append(self._birth(dets[high[k]], high[k]))
                unmatched = [r for r in range(len(pool)) if x[r] < 0]
            else:
                for k in high:
                    if gt(scores[k], nth, f64):
                        nxt.append(self._birth(dets[k], k))
        upool = [pool[r] for r in unmatched] if unmatched else []
        next_lost = list(upool)
        if mid and not unmatched:
            self._hit("pass2_skipped" if not high and pool else "pass2_none")
        if mid and unmatched:
            cost = cost_matrix([t.box for t in upool], dets[mid, :4], True).astype(np.float64)
            _, x, _ = lapjv(cost, extend_cost=True, cost_limit=c["match_th_second"])
            for r in range(len(upool)):
                if x[r] >= 0:
                    t = upool[r]
                    self._update(t, dets[mid[x[r]]], self.frame, mid[x[r]])
                    nxt.append(t)
                    self._hit("match_pass2")
                    if t in self.lost:
                        self.lost.remove(t)
                        self._hit("reacquire_pass2")
                    next_lost.remove(t)
        if not high and not mid:
            next_lost = list(pool)
            if pool:
                self._hit("all_to_lost")
        if mid and not high and self.active:
            self._hit("vanish")
        l, r_, t_, b = self.mrg if self.mrg is not None else (0.0, 0.0, 0.0, 0.0)
        for t in next_lost:
            if t not in self.lost:
                self.lost.append(t)
                u = t.box[0] + (t.box[2] - t.box[0]) / F32(2)
                v = t.box[1] + (t.box[3] - t.box[1]) / F32(2)
                central = F32(l) < u < F32(r_) and F32(t_) < v < F32(b)
                t.state = LOST_CENTRAL if central else LOST_MARGINAL
                self._hit("lost_central" if central else "lost_marginal")
        self.active = nxt
        if not nxt:
            return np.empty((0, 8), F32)
        return np.asarray([[*t.box, t.id, t.conf, t.cls, t.det_ind] for t in nxt], F32)

    def active_ids(self):
        return [t.id for t in self.active]

    def lost_ids(self):
        return [t.id for t in self.lost]

    def lost_states(self):
        return [t.state for t in self.lost]


def make(**kwargs) -> SfOracle:
    return SfOracle(resolve(**kwargs))


def load_case(name):
    """(per-frame rows, active ids, lost ids, lost states, (H, W)) of tests/golden/<name>.npz."""
    from tests.common import GOLDEN

    z = np.load(GOLDEN / f"{name}.npz")

    def split(a, off):
        return [a[off[i]:off[i + 1]] for i in range(len(off) - 1)]

    return (split(z["rows"], z["offsets"]), split(z["active"], z["act_off"]), split(z["lost"], z["lost_off"]),
            split(z["lost_state"], z["lost_off"]), tuple(int(v) for v in z["hw"]))

