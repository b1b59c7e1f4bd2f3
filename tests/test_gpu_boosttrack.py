"""BoostTrack / BoostTrack++ on the GPU (csrc/bt_core.cuh through the engine, the C ABI and `boxmot_b200.BoostTrack`)
against the goldens of the unmodified reference class and the oracle restatement (tests/boosttrack_oracle.py)."""
import numpy as np
import pytest

from tests.boosttrack_cases import CASES
from tests.common import assert_rows_match, load_golden

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


@pytest.mark.parametrize("name", sorted(CASES))
def test_boosttrack_goldens(name):
    import boxmot_b200 as bb

    kw = _kwargs(name)
    want, snaps = load_golden(name)
    frames, embs, warps = _inputs(name)
    trk = bb.BoostTrack(reid_model=_Model() if kw.get("with_reid") else None, use_cmc=False, cap_tracks=512,
                        cap_dets=320, **kw)
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


def test_multistream_equals_independent_trackers():
    import boxmot_b200 as bb

    names = ["boosttrackpp_stress96", "boosttrack_yaml_stress48_gaps", "boosttrack_warp_stress64"]
    ins = [_inputs(n) for n in names]
    kw = _kwargs(names[0])
    assert all(_kwargs(n) == kw for n in names)
    ms = bb.MultiStreamTracker("boosttrack", n_streams=3, cap_tracks=512, cap_dets=320, **kw)
    single = [bb.MultiStreamTracker("boosttrack", n_streams=1, cap_tracks=512, cap_dets=320, **kw) for _ in names]
    n = min(len(i[0]) for i in ins)
    for f in range(n):
        for s, (fr, em, wa) in enumerate(ins):
            if wa is not None:
                ms.set_warp(s, wa[f])
                single[s].set_warp(0, wa[f])
        got = ms.update([i[0][f] for i in ins], None, [i[1][f] for i in ins])
        for s, (fr, em, wa) in enumerate(ins):
            one = single[s].update([fr[f]], None, [em[f]])[0]
            assert np.array_equal(np.asarray(got[s]), np.asarray(one)), f"stream {s} frame {f}"


def test_device_path_and_pipeline_equal_update_batch(tmp_path):
    """update_device + fetch == update_batch (supplied embeddings); with on-device ReID the pipelined sync=False path
    equals the synchronous one."""
    import torch

    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_osnet_state
    from boxmot_b200.weights import export_blob

    kw = _kwargs("boosttrackpp_stress96")
    frames, embs, _ = _inputs("boosttrackpp_stress96")
    frames, embs = frames[:60], embs[:60]
    a = bb.MultiStreamTracker("boosttrack", 1, 512, 320, **kw)
    b = bb.MultiStreamTracker("boosttrack", 1, 512, 320, **kw)
    for d, e in zip(frames, embs):
        want = a.update([d], None, [e])[0]
        dd = torch.zeros((1, 320, 6), dtype=torch.float32, device="cuda")
        de = torch.zeros((1, 320, 512), dtype=torch.float32, device="cuda")
        dd[0, :len(d)] = torch.from_numpy(d)
        if len(d):
            de[0, :len(d)] = torch.from_numpy(e)
        b.update_device(dd, [len(d)], de)
        assert np.array_equal(np.asarray(b.fetch()[0]), np.asarray(want))

    img, fr = bench_stream(64, 12, hw=(360, 640))
    blob = export_blob(make_osnet_state("osnet_x0_25", seed=7), tmp_path / "m.b200reid")
    sync = bb.MultiStreamTracker("boosttrack", 1, 256, 128, reid_blob=str(blob), **kw)
    pipe = bb.MultiStreamTracker("boosttrack", 1, 256, 128, reid_blob=str(blob), **kw)
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
    """Frames in, ids out: every row cropped and embedded by OSNet_x0_25 on the device, the survivors' rows picked by
    the frame kernel; against the oracle BoostTrack++ fed by the oracle ReID (which embeds the survivors only)."""
    import boxmot_b200 as bb
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import bench_stream, make_osnet_state
    from boxmot_b200.weights import export_blob
    from oracle import reid as orid
    from tests.boosttrack_oracle import BoostTrackOracle

    img, frames = bench_stream(24, 10, hw=(360, 640))
    sd = make_osnet_state("osnet_x0_25", seed=7)
    reid = B200ReID(export_blob(sd, tmp_path / "m.b200reid"))
    kw = {k: v for k, v in _kwargs("boosttrackpp_stress96").items()}
    kw["det_thresh"] = 0.5
    gpu = bb.BoostTrack(reid_model=reid, use_cmc=False, cap_tracks=128, cap_dets=64, **kw)
    orc = BoostTrackOracle(reid_model=orid.OracleReID(sd), **kw)
    for f, d in enumerate(frames):
        got, want = gpu.update(d, img), orc.update(d, img)
        assert np.array_equal(np.asarray(got)[:, 4], np.asarray(want, np.float32)[:, 4]), f"frame {f}: ids"
        assert_rows_match(got, want, f)
    # a row's embedding does not depend on which other rows are embedded with it
    boxes = frames[3][:, :4]
    every = reid.get_features(boxes, img)
    keep = np.flatnonzero(frames[3][:, 4] >= 0.5)
    some = reid.get_features(boxes[keep], img)
    assert np.array_equal(every[keep], some)


@pytest.mark.parametrize("method", ["ecc", "sof"])
def test_device_cmc_equals_supplied_standalone_warps(method):
    import ctypes

    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import camera_pan_sequence

    frames, dets, _, _ = camera_pan_sequence(16, seed=11)
    kw = dict(_kwargs("boosttrack_stress96"), det_thresh=0.3)
    est = bb.BoostTrack(use_cmc=True, cmc_method=method, cap_tracks=128, cap_dets=64, **kw)
    fed = bb.BoostTrack(use_cmc=False, cap_tracks=128, cap_dets=64, **kw)
    lib = _lib.require_device()
    sof = bb.SOF() if method == "sof" else None
    h, w = frames[0].shape[:2]
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
        if f > 2:
            assert len(a) > 0


def test_reset_empty_frames_and_capacity_errors():
    import boxmot_b200 as bb

    frames, _, _ = _inputs("boosttrack_stress96")
    trk = bb.BoostTrack(use_cmc=False, cap_tracks=512, cap_dets=320)
    first = [np.asarray(trk.update(d, None)) for d in frames[:20]]
    assert trk.update(np.empty((0, 6), np.float32), None).shape == (0, 8)
    trk.reset()
    again = [np.asarray(trk.update(d, None)) for d in frames[:20]]
    assert all(np.array_equal(x, y) for x, y in zip(first, again))
    small = bb.BoostTrack(use_cmc=False, cap_tracks=8, cap_dets=320)
    with pytest.raises(bb.B200Error, match="track capacity"):
        for d in frames[:5]:
            small.update(d, None)
    with pytest.raises(bb.B200Error):   # sticky: the stream stays in error
        small.update(frames[5], None)
    tiny = bb.BoostTrack(use_cmc=False, cap_tracks=64, cap_dets=4)
    with pytest.raises(bb.B200Error, match="cap_dets"):
        tiny.update(frames[10], None)
