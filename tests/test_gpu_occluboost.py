"""OccluBoost on the GPU (csrc/ob_core.cuh through the engine, the C ABI and `boxmot_b200.OccluBoost`) against the
goldens of the unmodified reference class and the oracle restatement (tests/occluboost_oracle.py)."""
import numpy as np
import pytest

from tests.common import GOLDEN, assert_rows_match, load_golden
from tests.occluboost_cases import CASES

pytestmark = pytest.mark.gpu


class _Model:   # with_reid needs a model; embeddings are supplied, so it is never called
    def get_features(self, xyxys, img):
        raise AssertionError("embeddings are supplied")


def _kwargs(name):
    return {k: v for k, v in CASES[name][0].items() if k not in ("use_cmc", "cmc_method")}


def _inputs(name):
    _, make_frames, make_embs, make_warps = CASES[name]
    frames = make_frames()
    return frames, (make_embs(frames) if make_embs else None), (make_warps() if make_warps else None)


def _feat(embs):
    return 512 if embs is None else embs[0].shape[1]


@pytest.mark.parametrize("name", sorted(CASES))
def test_occluboost_goldens(name):
    import boxmot_b200 as bb

    kw = _kwargs(name)
    want, snaps = load_golden(name)
    z = np.load(GOLDEN / f"{name}.npz")
    frames, embs, warps = _inputs(name)
    trk = bb.OccluBoost(reid_model=_Model() if kw.get("with_reid") else None, use_cmc=False, cap_tracks=512,
                        cap_dets=320, feat_dim=_feat(embs), **kw)
    for f, d in enumerate(frames, start=1):
        got = trk.update(d, None, None if embs is None else embs[f - 1], warp=None if warps is None else warps[f - 1])
        assert_rows_match(got, want[f - 1], f)
        if f in snaps:
            ids, mean, cov = snaps[f]
            st = trk.snapshot()
            assert [v.id for v in trk.active_tracks] == ids.tolist(), f"frame {f}: track list"
            for i, tid in enumerate(ids):
                np.testing.assert_allclose(st[int(tid)][0], mean[i], rtol=1e-9, atol=1e-7)
                np.testing.assert_allclose(st[int(tid)][1], cov[i], rtol=1e-9, atol=1e-7)
    np.testing.assert_allclose(trk.flush_gta(), z["gta"], rtol=1e-9, atol=1e-6, err_msg="flush_gta rows")
    assert trk.flush_gta().shape == (0, 9)


def test_multistream_equals_independent_trackers():
    import boxmot_b200 as bb

    names = ["occluboost_ctor_stress96", "occluboost_gaps_stress48"]
    ins = [_inputs(n) for n in names]
    kw = dict(with_reid=True, use_second_pass=True)
    ms = bb.MultiStreamTracker("occluboost", n_streams=2, cap_tracks=512, cap_dets=320, **kw)
    single = [bb.MultiStreamTracker("occluboost", n_streams=1, cap_tracks=512, cap_dets=320, **kw) for _ in names]
    n = min(len(i[0]) for i in ins)
    for f in range(n):
        got = ms.update([i[0][f] for i in ins], None, [i[1][f] for i in ins])
        for s, (fr, em, _) in enumerate(ins):
            one = single[s].update([fr[f]], None, [em[f]])[0]
            assert np.array_equal(np.asarray(got[s]), np.asarray(one)), f"stream {s} frame {f}"
    for s in range(2):
        assert np.array_equal(ms.flush_gta(s), single[s].flush_gta(0))


def test_device_path_and_pipeline_equal_update_batch(tmp_path):
    """update_device + fetch == update_batch (supplied embeddings, GTA events taken at the end); with on-device ReID the
    pipelined sync=False path equals the synchronous one."""
    import torch

    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_osnet_state
    from boxmot_b200.weights import export_blob

    kw = _kwargs("occluboost_gta24")
    frames, embs, _ = _inputs("occluboost_gta24")
    F = _feat(embs)
    a = bb.MultiStreamTracker("occluboost", 1, 512, 320, feat_dim=F, **kw)
    b = bb.MultiStreamTracker("occluboost", 1, 512, 320, feat_dim=F, **kw)
    for d, e in zip(frames, embs):
        want = a.update([d], None, [e])[0]
        dd = torch.zeros((1, 320, 6), dtype=torch.float32, device="cuda")
        de = torch.zeros((1, 320, F), dtype=torch.float32, device="cuda")
        dd[0, :len(d)] = torch.from_numpy(d)
        if len(d):
            de[0, :len(d)] = torch.from_numpy(e)
        b.update_device(dd, [len(d)], de)
        assert np.array_equal(np.asarray(b.fetch()[0]), np.asarray(want))
    ga = a.flush_gta(0)
    assert len(ga) > 100 and np.array_equal(ga, b.flush_gta(0))

    kw = _kwargs("occluboost_yaml_stress96")
    img, fr = bench_stream(64, 12, hw=(360, 640))
    blob = export_blob(make_osnet_state("osnet_x0_25", seed=7), tmp_path / "m.b200reid")
    sync = bb.MultiStreamTracker("occluboost", 1, 256, 128, reid_blob=str(blob), **kw)
    pipe = bb.MultiStreamTracker("occluboost", 1, 256, 128, reid_blob=str(blob), **kw)
    dimg = torch.from_numpy(img).cuda().unsqueeze(0).contiguous()
    outs_s, outs_p = [], []
    for d in fr:
        dd = torch.zeros((1, 128, 6), dtype=torch.float32, device="cuda")
        dd[0, :len(d)] = torch.from_numpy(d)
        sync.update_device(dd, [len(d)], None, dimg, sync=True)
        outs_s.append(np.asarray(sync.fetch()[0]))
        pipe.update_device(dd, [len(d)], None, dimg, sync=False)
        outs_p.append(np.asarray(pipe.fetch()[0]))
    for f, (x, y) in enumerate(zip(outs_s, outs_p)):
        assert np.array_equal(x, y), f"frame {f}"
    assert sum(len(o) for o in outs_s) > 100


def test_on_device_reid_matches_the_oracle_with_the_oracle_reid(tmp_path):
    """Frames in, ids out: every row cropped and embedded by OSNet_x0_25 on the device; against the oracle OccluBoost fed
    by the oracle ReID."""
    import boxmot_b200 as bb
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import bench_stream, make_osnet_state
    from boxmot_b200.weights import export_blob
    from oracle import reid as orid
    from tests.occluboost_oracle import OccluBoostOracle

    img, frames = bench_stream(24, 10, hw=(360, 640))
    sd = make_osnet_state("osnet_x0_25", seed=7)
    reid = B200ReID(export_blob(sd, tmp_path / "m.b200reid"))
    kw = _kwargs("occluboost_yaml_stress96")
    gpu = bb.OccluBoost(reid_model=reid, use_cmc=False, cap_tracks=128, cap_dets=64, **kw)
    orc = OccluBoostOracle(reid_model=orid.OracleReID(sd), **kw)
    for f, d in enumerate(frames):
        got, want = gpu.update(d, img), orc.update(d, img)
        assert np.array_equal(np.asarray(got)[:, 4], np.asarray(want, np.float32)[:, 4]), f"frame {f}: ids"
        assert_rows_match(got, want, f)


@pytest.mark.parametrize("method", ["ecc", "sof"])
def test_device_cmc_equals_supplied_standalone_warps(method):
    import ctypes

    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import camera_pan_sequence

    frames, dets, _, _ = camera_pan_sequence(16, seed=11)
    kw = dict(_kwargs("occluboost_noreid_stress64"), det_thresh=0.3, new_track_thresh=0.3)
    est = bb.OccluBoost(use_cmc=True, cmc_method=method, cap_tracks=128, cap_dets=64, **kw)
    fed = bb.OccluBoost(use_cmc=False, cap_tracks=128, cap_dets=64, **kw)
    lib = _lib.require_device()
    sof = bb.SOF() if method == "sof" else None
    h, w = frames[0].shape[:2]
    n_rows = 0
    for f, (img, d) in enumerate(zip(frames, dets)):
        if method == "sof":
            warp = np.asarray(sof.apply(img, d), np.float64)
        elif f == 0:
            warp = np.eye(2, 3)
        else:
            w6 = np.zeros(6, np.float32)
            st = ctypes.c_int(0)
            assert lib.boxmot_b200_cmc_ecc(np.ascontiguousarray(frames[f - 1]).ctypes.data,
                                           np.ascontiguousarray(img).ctypes.data, h, w, 0.15, 1e-5, 100,
                                           w6.ctypes.data, ctypes.byref(st), None)
            warp = w6.astype(np.float64).reshape(2, 3)
        a, b = est.update(d, img), fed.update(d, img, warp=warp)
        assert np.array_equal(np.asarray(a), np.asarray(b)), f"frame {f}"
        n_rows += len(a)
    assert n_rows > 0


def test_reset_empty_frames_and_capacity_errors():
    import boxmot_b200 as bb
    from oracle.streams import stress_stream, unit_embeddings

    name = "occluboost_gta24"
    frames, embs, _ = _inputs(name)
    kw = _kwargs(name)
    trk = bb.OccluBoost(reid_model=_Model(), use_cmc=False, cap_tracks=512, cap_dets=320, feat_dim=128, **kw)
    first = [np.asarray(trk.update(d, None, e)) for d, e in zip(frames[:120], embs[:120])]
    assert trk.update(np.empty((0, 6), np.float32), None).shape == (0, 8)
    trk.reset()   # graveyard and pending gap rows go too
    assert trk.flush_gta().shape == (0, 9)
    again = [np.asarray(trk.update(d, None, e)) for d, e in zip(frames[:120], embs[:120])]
    assert all(np.array_equal(x, y) for x, y in zip(first, again))
    small = bb.OccluBoost(use_cmc=False, cap_tracks=8, cap_dets=320, new_track_thresh=0.1)
    with pytest.raises(bb.B200Error, match="track capacity"):
        for d in stress_stream(96, 5):
            small.update(d, None)
    tiny = bb.OccluBoost(use_cmc=False, cap_tracks=64, cap_dets=4)
    with pytest.raises(bb.B200Error, match="cap_dets"):
        tiny.update(stress_stream(96, 12)[10], None)
    # graveyard overflow: every track dies after one missed frame and stays buried, the live tracks always fit
    fr = stress_stream(96, 60, seed=5)
    em = unit_embeddings(fr, 96, seed=5)
    grave = bb.OccluBoost(reid_model=_Model(), with_reid=True, use_cmc=False, cap_tracks=128, cap_dets=128, max_age=0,
                          gta_min_track_length=1, gta_max_gap=1000, gta_appearance_thresh=0.99)
    with pytest.raises(bb.B200Error, match="track capacity"):
        for d, e in zip(fr, em):
            grave.update(d, None, e)


def test_replay_appends_the_flushed_gap_rows(tmp_path):
    import boxmot_b200 as bb
    from boxmot_b200.replay import SequenceCache, replay_sequences, to_mot_rows, write_cache

    kw = _kwargs("occluboost_gta24")
    frames, embs, _ = _inputs("occluboost_gta24")
    write_cache(tmp_path / "d.npy", tmp_path / "e.npy", [(i + 1, d, e) for i, (d, e) in enumerate(zip(frames, embs))
                                                         if len(d)])
    cache = SequenceCache(str(tmp_path / "d.npy"), str(tmp_path / "e.npy"))
    ms = bb.MultiStreamTracker("occluboost", 1, 512, 320, feat_dim=128, **kw)
    got = replay_sequences(ms, [cache])[0]
    ref = bb.MultiStreamTracker("occluboost", 1, 512, 320, feat_dim=128, **kw)
    rows = [to_mot_rows(np.asarray(ref.update([d], None, [e])[0]), i + 1) for i, (d, e) in enumerate(zip(frames, embs))
            if len(d)]
    gta = ref.flush_gta(0)
    assert len(gta) > 100
    want = np.concatenate([r for r in rows if len(r)] + [gta.astype(np.float32)], 0)
    assert np.array_equal(got, want)
