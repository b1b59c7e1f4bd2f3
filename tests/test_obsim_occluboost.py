"""The OccluBoost device core (boxmot_b200/csrc/ob_core.cuh) compiled for the host (tests/obsim.py) against every golden
of the unmodified reference class: ids, det_ind, cls and conf exact, boxes within the row tolerance, Kalman snapshots
and is_activated, the resurrection events equal to the oracle's, and flush_gta() rows rebuilt from them.  Also the AMS
gain factor of the device source against numpy on random buffers."""
from collections import deque

import numpy as np
import pytest

from boxmot_b200.trackers import gta_rows
from tests.common import GOLDEN, assert_rows_match, load_golden
from tests.obsim import ObSimTracker, lib, make_cfg
from tests.occluboost_cases import CASES
from tests.occluboost_oracle import OB_DEFAULTS, OccluBoostOracle


def sim_kwargs(kwargs):
    return {k: v for k, v in kwargs.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_build_of_the_device_core_matches_the_reference(name):
    kwargs, make_frames, make_embs, make_warps = CASES[name]
    want, snaps = load_golden(name)
    z = np.load(GOLDEN / f"{name}.npz")
    frames = make_frames()
    embs = make_embs(frames) if make_embs else None
    warps = make_warps() if make_warps else None
    kw = sim_kwargs(kwargs)
    feat = embs[0].shape[1] if embs is not None else 512
    trk = ObSimTracker(make_cfg(feat_dim=feat, **kw))
    events = []
    for f, d in enumerate(frames, start=1):
        got = trk.update(d, None if embs is None else embs[f - 1], None if warps is None else warps[f - 1])
        assert_rows_match(got, want[f - 1], f)
        events.append(trk.take_events())
        if f in snaps:
            ids, mean, cov = snaps[f]
            gi, gx, gp, ga = trk.snapshot()
            assert gi.tolist() == ids.tolist(), f"frame {f}: track list"
            assert ga.tolist() == z[f"snap{f}_act"].tolist(), f"frame {f}: is_activated"
            np.testing.assert_allclose(gx, mean, rtol=1e-9, atol=1e-7, err_msg=f"frame {f}: means")
            np.testing.assert_allclose(gp, cov, rtol=1e-9, atol=1e-7, err_msg=f"frame {f}: covariances")
    o = dict(OB_DEFAULTS, **{k: v for k, v in kw.items() if k in OB_DEFAULTS})
    ev = np.concatenate(events, 0)
    rows = gta_rows(ev, o["gta_interpolate"], max(int(o["gta_max_gap"]), 1), o["gta_smooth_tau"])
    np.testing.assert_allclose(rows, z["gta"], rtol=1e-9, atol=1e-6, err_msg="flush_gta rows")


def test_gta_events_equal_the_oracle():
    kwargs, make_frames, make_embs, _ = CASES["occluboost_gta24"]
    frames = make_frames()
    embs = make_embs(frames)

    class _Model:
        pass

    o = OccluBoostOracle(reid_model=_Model(), **kwargs)
    trk = ObSimTracker(make_cfg(feat_dim=embs[0].shape[1], **kwargs))
    n = 0
    for f, d in enumerate(frames):
        before = len(o.gap_rows)
        o.update(d.copy(), None, embs[f])
        trk.update(d, embs[f])
        ev = trk.take_events()
        for e in ev:   # each event expands to the oracle's rows of that resurrection, in order
            gap = int(e[2] - e[1])
            for k in range(1, gap):
                a = k / gap
                row = o.gap_rows[before]
                before += 1
                assert row[0] == e[1] + k and row[1] == e[0]
                np.testing.assert_allclose(row[2:6], (1.0 - a) * e[3:7] + a * e[7:11], rtol=0, atol=1e-9)
                # conf is the boosted float64 confidence: the soft-BIoU boost's x ** 1.5 may differ from numpy's power
                # in the last bit (invisible in the float32 output rows)
                np.testing.assert_allclose(row[6:8], e[11:13], rtol=1e-12, atol=0)
            n += 1
        assert before == len(o.gap_rows), f"frame {f + 1}: the oracle logged more gap rows"
    assert n >= 5


def test_ams_alpha_matches_numpy():
    h = lib()
    rng = np.random.default_rng(3)
    for case in range(30000):
        B = int(rng.integers(2, 61))
        n = int(rng.integers(0, B + 1))
        scale = float(rng.choice([1.0, 10.0, 100.0]))
        obs = np.empty((n, 4))
        obs[:, :2] = rng.uniform(0, 600, (n, 2))
        obs[:, 2:] = rng.uniform(5, 120, (n, 2))
        if n:
            obs = obs + rng.normal(0, 1, (n, 4)) * rng.uniform(0, 1) * scale * 0.01
        box = np.array([*rng.uniform(0, 600, 2), 0, 0])
        box[2:] = box[:2] + rng.uniform(1, 150, 2)
        a0, thr, shrink = float(rng.uniform(0, 1)), float(rng.uniform(0, 1)), float(rng.uniform(0.5, 1.0))
        # numpy, as occluboost.py:778-844
        buf = deque((r.copy() for r in obs), maxlen=B)
        x1, y1, x2, y2 = map(float, box)
        w, hh = max(x2 - x1, 1e-6), max(y2 - y1, 1e-6)
        cur = np.array([x1 + 0.5 * w, y1 + 0.5 * hh, w, hh])
        if len(buf) < 2:
            want = 1.0
        else:
            cv = cur - buf[-1]
            mv = np.diff(np.asarray(buf, dtype=float), axis=0).mean(axis=0)
            d_c = max(0.0, float(np.linalg.norm(cv[:2])) - float(np.linalg.norm(mv[:2]))) / max(float(np.linalg.norm(mv[:2])), 1e-6)
            d_a = max(0.0, float(np.linalg.norm(cv[2:])) - float(np.linalg.norm(mv[2:]))) / max(float(np.linalg.norm(mv[2:])), 1e-6)
            want = 0.5 * ((1.0 if d_c <= thr else a0) + (1.0 if d_a <= thr else a0))
            if float(cur[2] * cur[3]) >= float(np.mean(np.asarray(buf, dtype=float)[:, 2:].prod(axis=1))) * shrink:
                want = 1.0
        o = np.ascontiguousarray(obs)
        got = h.obsim_ams_alpha(o.ctypes.data, n, B, np.ascontiguousarray(box).ctypes.data, a0, thr, shrink)
        assert got == want, f"case {case}: {got} vs {want}"
