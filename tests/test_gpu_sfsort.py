"""SFSORT on the H100 against the reference goldens (tests/golden/sfsort_*.npz): rows, active ids and lost ids bit-exact
through `SFSORT.update`, through the reference-named C ABI `boxmot_sfsort_*` (constructor clamps included), and with
distinct golden streams in one `MultiStreamTracker` (synchronous and device-resident); streams and replayed sequences of
different resolutions against the oracle fed each one's frame size; reset, empty frames, the sticky capacity error and
the refused camera-motion calls."""
import ctypes

import numpy as np
import pytest

from tests import sfsort_oracle as so
from tests.sfsort_cases import CASES

pytestmark = pytest.mark.gpu
NAMES = sorted(CASES)


def _check(name, update, ids=None):
    kwargs, make_frames, hw = CASES[name]
    rows, act, lost, _, _ = so.load_case(name)
    for f, d in enumerate(make_frames()):
        out = np.asarray(update(d, hw), np.float32).reshape(-1, 8)
        assert np.array_equal(out, rows[f]), f"{name} frame {f}"
        if ids is not None:
            assert ids(0) == act[f].tolist() and ids(1) == lost[f].tolist(), f"{name} frame {f}"


@pytest.mark.parametrize("name", NAMES)
def test_class_matches_golden(name):
    import boxmot_b200 as bb

    t = bb.SFSORT(cap_tracks=1024, cap_dets=512, **CASES[name][0])
    _check(name, lambda d, hw: t.update(d, np.zeros((hw[0], hw[1], 3), np.uint8)), t._engine.track_ids)
    assert [v.id for v in t.lost_tracks] == t._engine.track_ids(1)


@pytest.mark.parametrize("name", NAMES)
def test_reference_c_abi_matches_golden(name):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    r = so.resolve(**CASES[name][0])
    c = _lib.BoxMOTSFSORTConfig(frame_rate=30, max_obs=50, obb_theta_damping=0.8,
                                frame_width=r["frame_width"] or 0, frame_height=r["frame_height"] or 0,
                                horizontal_margin=int(r["horizontal_margin"]), vertical_margin=int(r["vertical_margin"]),
                                dynamic_tuning=int(r["dynamic_tuning"]), marginal_timeout=r["marginal_timeout"],
                                central_timeout=r["central_timeout"],
                                **{k: r[k] for k in ("high_th", "match_th_first", "new_track_th", "low_th", "match_th_second",
                                                     "cth", "high_th_m", "new_track_th_m", "match_th_first_m")})
    h = lib.boxmot_sfsort_create(ctypes.byref(c))
    assert h, lib.boxmot_sfsort_last_error()
    try:
        def upd(d, hw):
            d = np.ascontiguousarray(d, np.float32)
            out = np.zeros((max(len(d), 1), 9), np.float32)
            n, obb = ctypes.c_int(0), ctypes.c_int(7)
            img = np.zeros((hw[0], hw[1], 3), np.uint8)
            ok = lib.boxmot_sfsort_update(h, d.ctypes.data if len(d) else None, len(d), 6, img.ctypes.data, hw[0], hw[1],
                                          3, out.ctypes.data, len(out), 9, ctypes.byref(n), ctypes.byref(obb))
            assert ok, lib.boxmot_sfsort_last_error()
            assert obb.value == 0
            return out[: n.value, :8]

        _check(name, upd)
        d7 = np.zeros((1, 7), np.float32)
        out = np.zeros((1, 9), np.float32)
        n, obb = ctypes.c_int(0), ctypes.c_int(0)
        assert not lib.boxmot_sfsort_update(h, d7.ctypes.data, 1, 7, None, 0, 0, 3, out.ctypes.data, 1, 9,
                                            ctypes.byref(n), ctypes.byref(obb))
        assert b"OBB" in lib.boxmot_sfsort_last_error()
        assert lib.boxmot_sfsort_reset(h)
    finally:
        lib.boxmot_sfsort_destroy(h)


def _multi(names, device):
    """Distinct golden streams that resolve to one configuration, each with its own frame size, in one handle."""
    import torch

    import boxmot_b200 as bb

    S, CD = len(names), 512
    kw = CASES[names[0]][0]
    assert all(so.resolve(**CASES[n][0]) == so.resolve(**kw) for n in names)
    hws = [CASES[n][2] for n in names]
    m = bb.MultiStreamTracker("sfsort", n_streams=S, cap_tracks=1024, cap_dets=CD, **kw)
    streams = [CASES[n][1]() for n in names]
    golds = [so.load_case(n) for n in names]
    n_frames = min(len(s) for s in streams)
    imgs = [np.zeros((hw[0], hw[1], 3), np.uint8) for hw in hws]
    for f in range(n_frames):
        dets = [s[f] for s in streams]
        if device:
            buf = np.zeros((S, CD, 6), np.float32)
            for i, d in enumerate(dets):
                buf[i, : len(d)] = d
            m.update_device(torch.from_numpy(buf).cuda(), [len(d) for d in dets], image_hw=hws, sync=False)
            outs = m.fetch()
        else:
            outs = m.update(dets, imgs)
        for i in range(S):
            assert np.array_equal(np.asarray(outs[i]), golds[i][0][f]), f"stream {i} frame {f}"
            assert m.track_ids(0, i) == golds[i][1][f].tolist(), f"stream {i} frame {f}"
            assert m.track_ids(1, i) == golds[i][2][f].tolist(), f"stream {i} frame {f}"


def test_multistream_equals_independent_trackers():
    _multi(["sfsort_ctor_stress96", "sfsort_yaml_stress64"], False)
    _multi(["sfsort_timeouts_stress64", "sfsort_duplicates_stress32"], False)


def test_update_device_and_fetch():
    _multi(["sfsort_duplicates_stress32", "sfsort_timeouts_stress64"], True)


# unequal timeouts: a lost track's central / marginal state, decided by its stream's margins, decides when it is purged
KW_MIXED = dict(central_timeout=12, marginal_timeout=4, horizontal_margin=60, vertical_margin=40)
HWS = [(360, 640), (1080, 1920)]


def _mixed_streams():
    from oracle.streams import stress_stream

    return [stress_stream(48, 100, seed=61, empty_every=23), stress_stream(48, 100, seed=62, empty_every=29)]


def _oracle_rows(frames, hw):
    o = so.make(**KW_MIXED)
    rows, lost = [], []
    for d in frames:
        rows.append(o.update(d, hw))
        lost.append(o.lost_ids())
    return rows, lost


def test_streams_of_different_resolution_keep_their_own_margins():
    import torch

    import boxmot_b200 as bb

    streams = _mixed_streams()
    want = [_oracle_rows(fr, hw) for fr, hw in zip(streams, HWS)]
    # the resolution matters for this stream: fed the other stream's frame size it tracks differently
    other = _oracle_rows(streams[1], HWS[0])
    assert any(len(a) != len(b) or not np.array_equal(a, b) for a, b in zip(want[1][0], other[0]))
    assert want[1][1] != other[1]
    for device in (False, True):
        m = bb.MultiStreamTracker("sfsort", n_streams=2, cap_tracks=512, cap_dets=256, **KW_MIXED)
        imgs = [np.zeros((h, w, 3), np.uint8) for h, w in HWS]
        for f in range(len(streams[0])):
            dets = [s[f] for s in streams]
            if device:
                buf = np.zeros((2, 256, 6), np.float32)
                for i, d in enumerate(dets):
                    buf[i, : len(d)] = d
                m.update_device(torch.from_numpy(buf).cuda(), [len(d) for d in dets], image_hw=HWS)
                outs = m.fetch()
            else:
                outs = m.update(dets, imgs)
            for i in range(2):
                assert np.array_equal(np.asarray(outs[i]), want[i][0][f]), f"device={device} stream {i} frame {f}"
                assert m.track_ids(1, i) == want[i][1][f], f"device={device} stream {i} frame {f}"


def test_margins_that_matter_need_a_frame_size():
    import boxmot_b200 as bb

    m = bb.MultiStreamTracker("sfsort", n_streams=2, cap_tracks=64, cap_dets=64, **KW_MIXED)
    d = [np.zeros((0, 6), np.float32)] * 2
    with pytest.raises(bb.B200Error, match="no frame size"):
        m.update(d, None)
    m.set_frame_size(0, HWS[0])
    with pytest.raises(bb.B200Error, match="stream 1 has no frame size"):
        m.update(d, None)
    m.set_frame_size(1, HWS[1])
    m.update(d, None)
    # equal timeouts or margins from frame_width / frame_height: no frame needed
    bb.MultiStreamTracker("sfsort", n_streams=1, cap_tracks=64, cap_dets=64).update(d[:1], None)
    bb.MultiStreamTracker("sfsort", n_streams=1, cap_tracks=64, cap_dets=64, frame_width=640, frame_height=360,
                          **KW_MIXED).update(d[:1], None)
    with pytest.raises(bb.B200Error, match="SFSORT"):
        bb.MultiStreamTracker("bytetrack", n_streams=1, cap_tracks=64, cap_dets=64).set_frame_size(0, HWS[0])


def test_constructor_clamps_through_the_c_abi():
    """Out-of-range arguments through boxmot_sfsort_create are clamped as the reference's constructor clamps them
    (tests/golden/sfsort_contract.json pins the oracle's clamps)."""
    import json

    from boxmot_b200 import _lib
    from oracle.streams import stress_stream
    from tests.common import GOLDEN

    lib = _lib.require_device()
    frames = stress_stream(48, 80, seed=3, empty_every=17)
    hw = (360, 640)
    for case in json.loads((GOLDEN / "sfsort_contract.json").read_text())["resolved"]:
        args = {k: v for k, v in case["args"].items() if v is not None}
        full = dict(high_th=0.6, match_th_first=0.67, new_track_th=0.7, low_th=0.1, match_th_second=0.3, cth=0.5,
                    high_th_m=0.0, new_track_th_m=0.0, match_th_first_m=0.0, central_timeout=5, marginal_timeout=2,
                    horizontal_margin=30, vertical_margin=20)
        full.update({k: v for k, v in args.items() if k != "dynamic_tuning"})
        c = _lib.BoxMOTSFSORTConfig(dynamic_tuning=int(bool(args.get("dynamic_tuning"))), frame_rate=30, max_obs=50,
                                    obb_theta_damping=0.8, **full)
        o = so.make(dynamic_tuning=bool(args.get("dynamic_tuning")), **full)
        h = lib.boxmot_sfsort_create(ctypes.byref(c))
        assert h, lib.boxmot_sfsort_last_error()
        try:
            img = np.zeros((hw[0], hw[1], 3), np.uint8)
            for f, d in enumerate(frames):
                d = np.ascontiguousarray(d, np.float32)
                out = np.zeros((max(len(d), 1), 9), np.float32)
                n, obb = ctypes.c_int(0), ctypes.c_int(0)
                assert lib.boxmot_sfsort_update(h, d.ctypes.data if len(d) else None, len(d), 6, img.ctypes.data, hw[0],
                                                hw[1], 3, out.ctypes.data, len(out), 9, ctypes.byref(n), ctypes.byref(obb))
                assert np.array_equal(out[: n.value, :8], o.update(d, hw)), f"{case['args']} frame {f}"
        finally:
            lib.boxmot_sfsort_destroy(h)


def test_ignored_constructor_arguments():
    import boxmot_b200 as bb

    t = bb.SFSORT(asso_func="giou", obb_theta_damping=3.0, cap_tracks=64, cap_dets=64)
    assert t.obb_theta_damping == 1.0 and t.asso_func_name == "giou"


def test_reset_empty_frames_and_refusals():
    import boxmot_b200 as bb

    t = bb.SFSORT(cap_tracks=64, cap_dets=64)
    img = np.zeros((360, 640, 3), np.uint8)
    assert t.update(np.empty((0, 6), np.float32), img).shape == (0, 8)
    d = np.array([[10, 10, 50, 90, 0.9, 0], [100, 20, 140, 120, 0.8, 1]], np.float32)
    assert t.update(d, img)[:, 4].tolist() == [0, 1]
    assert t.update(np.empty((0, 6), np.float32), img).shape == (0, 8)
    t.reset()
    assert t.update(d[::-1].copy(), img)[:, 4].tolist() == [0, 1]
    with pytest.raises(bb.B200Error):
        t.set_cmc("ecc")
    with pytest.raises(bb.B200Error):
        t._engine.set_warp(0, np.eye(2, 3))
    with pytest.raises(NotImplementedError):
        t.update(np.zeros((1, 7), np.float32), img)


def test_capacity_error_is_sticky_and_cleared_by_reset():
    import boxmot_b200 as bb

    t = bb.SFSORT(cap_tracks=8, cap_dets=32)
    img = np.zeros((360, 640, 3), np.uint8)
    dets = np.array([[10 * k, 10, 10 * k + 8, 30, 0.9, 0] for k in range(12)], np.float32)
    with pytest.raises(bb.B200Error, match="cap_tracks"):
        t.update(dets, img)
    with pytest.raises(bb.B200Error, match="cap_tracks"):
        t.update(dets[:2], img)
    t.reset()
    assert t.update(dets[:2], img)[:, 4].tolist() == [0, 1]


def test_replay_two_sequences():
    """Two cached sequences of different resolution with unequal timeouts: full rows and lost ids per sequence equal
    the oracle fed that sequence's frame size; without the frame sizes replay refuses."""
    import boxmot_b200 as bb
    from boxmot_b200.replay import SequenceCache, replay_sequences, to_mot_rows

    streams = _mixed_streams()
    caches, want = [], []
    steps = max(sum(1 for d in fr if len(d)) for fr in streams)   # a finished sequence's stream gets empty frames
    for i, (fr, hw) in enumerate(zip(streams, HWS)):
        rows = [np.concatenate([np.full((len(d), 1), f + 1, np.float32), d], 1) for f, d in enumerate(fr) if len(d)]
        caches.append(SequenceCache(np.concatenate(rows, 0), name=f"seq{i}", frame_hw=hw))
        o = so.make(**KW_MIXED)
        mot = [to_mot_rows(o.update(d, hw), f + 1) for f, d in enumerate(fr) if len(d)]   # empty frames are skipped
        for _ in range(steps - len(mot)):
            o.update(np.zeros((0, 6), np.float32), hw)
        want.append((np.concatenate([r for r in mot if len(r)], 0), o.lost_ids()))
    m = bb.MultiStreamTracker("sfsort", n_streams=2, cap_tracks=512, cap_dets=256, **KW_MIXED)
    out = replay_sequences(m, caches)
    for i in range(2):
        assert np.array_equal(np.asarray(out[i], np.float32), np.asarray(want[i][0], np.float32)), f"sequence {i}"
        assert m.track_ids(1, i) == want[i][1], f"sequence {i}"
    bare = [SequenceCache(c.dets, name=c.name) for c in caches]
    with pytest.raises(bb.B200Error, match="no frame size"):
        replay_sequences(bb.MultiStreamTracker("sfsort", n_streams=2, cap_tracks=512, cap_dets=256, **KW_MIXED), bare)
