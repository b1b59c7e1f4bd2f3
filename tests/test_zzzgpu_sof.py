"""The SOF camera-motion estimator on the device (boxmot_b200.SOF, boxmot_b200_cmc_sof_*): bit for bit against the host
build of the same header (tests/sofsim.py), and within the CPU bounds of the cv2 restatement (tests/sof_oracle.py).
Sorts after the other GPU files so the newest kernels run last."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

from boxmot_b200.synthetic import camera_similarity_sequence  # noqa: E402
from tests import sofsim  # noqa: E402
from tests.sof_oracle import SofOracle  # noqa: E402


def _run(seq, **kw):
    import boxmot_b200 as bb

    dev, host, orc = bb.SOF(**kw), sofsim.HostSOF(**kw), SofOracle(**kw)
    statuses = []
    for f, (im, d) in enumerate(seq):
        got, want, ref = dev.apply(im, d), host.apply(im, d), orc.apply(im, d)
        assert dev.last_status == host.status == orc.status, f
        assert got.dtype == np.float32 and got.shape == (2, 3)
        np.testing.assert_array_equal(got, want, err_msg=f"frame {f}: device != host build")
        np.testing.assert_allclose(got[:, :2], ref[:, :2], rtol=0, atol=1e-4)
        np.testing.assert_allclose(got[:, 2], ref[:, 2], rtol=0, atol=0.02)
        statuses.append(dev.last_status)
    return statuses


@pytest.mark.parametrize("hw,seed", [((360, 640), 61), ((720, 1280), 62), ((1080, 1920), 63), ((475, 801), 64)])
def test_device_sof_matches_host_build_and_oracle(hw, seed):
    frames, dets, _ = camera_similarity_sequence(6, hw=hw, seed=seed)
    st = _run(zip(frames, dets))
    assert st[0] == 0 and st.count(1) >= 4


@pytest.mark.parametrize("kind", ["constant", "covered", "inverted", "few_inliers", "empty_dets"])
def test_device_sof_failure_paths(kind):
    frames, dets, _ = camera_similarity_sequence(5, hw=(360, 640), seed=65)
    seq = list(zip(frames, dets))
    kw = dict(min_inliers=5000) if kind == "few_inliers" else {}
    if kind == "constant":
        seq.insert(2, (np.full_like(frames[0], 128), dets[0]))
    elif kind == "covered":
        seq.insert(1, (frames[1], np.array([[-10, -10, 700, 400]], np.float32)))
    elif kind == "inverted":
        seq.insert(2, (255 - frames[1], dets[1]))
    elif kind == "empty_dets":
        seq = [(f, d[:0]) for f, d in seq]
    st = _run(seq, **kw)
    print(kind, st)


def test_device_sof_resolution_change_starts_afresh():
    a, da, _ = camera_similarity_sequence(3, hw=(360, 640), seed=66)
    b, db, _ = camera_similarity_sequence(3, hw=(720, 1280), seed=67)
    import boxmot_b200 as bb

    dev, host = bb.SOF(), sofsim.HostSOF()
    seen = []
    for im, d in list(zip(a, da)) + list(zip(b, db)) + list(zip(a, da)):
        np.testing.assert_array_equal(dev.apply(im, d), host.apply(im, d))
        assert dev.last_status == host.status
        seen.append(dev.last_status)
    assert seen[0] == seen[3] == seen[6] == 0


def test_c_abi_rejects_bad_arguments():
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    assert not lib.boxmot_b200_cmc_sof_create(0.0, 8, 0.2, 3.0)
    h = lib.boxmot_b200_cmc_sof_create(0.15, 8, 0.2, 3.0)
    assert h
    img = np.zeros((10, 10, 3), np.uint8)
    w = np.zeros(6, np.float32)
    st = ctypes.c_int(-1)
    assert lib.boxmot_b200_cmc_sof_apply(h, img.ctypes.data, 10, 10, None, 0, w.ctypes.data, ctypes.byref(st)) == 0
    assert "3x3" in _lib.last_error(lib)
    lib.boxmot_b200_cmc_sof_destroy(h)


# ---- SOF inside the trackers (set_cmc("sof"), DeepOcSort(cmc_off=False)) ------------------------------------------
BOT_KW = dict(with_reid=False, track_high_thresh=0.6, new_track_thresh=0.65)
DOC_KW = dict(embedding_off=True, det_thresh=0.7)


def _seq_with_gaps(n, hw, seed):
    frames, dets, _ = camera_similarity_sequence(n, hw=hw, seed=seed)
    return [(im, d[:0] if f in (7, 8) else d) for f, (im, d) in enumerate(zip(frames, dets))]   # two empty frames


def _est(status):
    return status == 1


def _check_tracker_against_oracles(gpu, make_oracle, seq, mask_rows):
    """The tracker's own SOF against (a) the oracle tracker fed the warps of the device's standalone SOF on the same
    frames and masked rows (ids exact, boxes 1e-4) and (b) the oracle tracker fed SofOracle's warps (boxes rtol 1e-3)."""
    import boxmot_b200 as bb
    from tests.common import assert_rows_match

    sof, ref = bb.SOF(), SofOracle()
    orc_dev, orc_cv = make_oracle(), make_oracle()
    moved = 0
    for f, (im, d) in enumerate(seq):
        w_dev = sof.apply(im, mask_rows(d))
        w_ref = ref.apply(im, mask_rows(d))
        moved += _est(sof.last_status)
        got = gpu.update(d, im)
        assert_rows_match(got, orc_dev.update(d, im, warp=w_dev if _est(sof.last_status) else None), f)
        assert_rows_match(got, orc_cv.update(d, im, warp=w_ref if _est(ref.status) else None), f, box_rtol=1e-3)
    assert moved >= len(seq) - 4
    return sof


def test_botsort_set_cmc_sof_matches_oracle():
    import boxmot_b200 as bb
    from oracle.trackers import BotSortOracle

    gpu = bb.BotSort(cap_tracks=128, cap_dets=64, **BOT_KW)
    gpu.set_cmc("sof")
    seq = _seq_with_gaps(20, (360, 640), 81)
    _check_tracker_against_oracles(gpu, lambda: BotSortOracle(**BOT_KW), seq, lambda d: d)
    gpu.reset()   # a fresh tracker with a fresh estimator
    _check_tracker_against_oracles(gpu, lambda: BotSortOracle(**BOT_KW), seq[:6], lambda d: d)
    with pytest.raises(NotImplementedError):
        bb.BotSort(use_cmc=True, cmc_method="sof", with_reid=False)


def test_deepocsort_cmc_on_matches_oracle():
    import boxmot_b200 as bb
    from oracle.deepocsort import DeepOcSortOracle

    gpu = bb.DeepOcSort(cmc_off=False, cap_tracks=128, cap_dets=64, **DOC_KW)
    seq = _seq_with_gaps(20, (360, 640), 82)
    keep = lambda d: d[d[:, 4] > np.float32(DOC_KW["det_thresh"])]   # noqa: E731  deepocsort.py:330-347
    assert any(0 < len(keep(d)) < len(d) for _, d in seq)
    _check_tracker_against_oracles(gpu, lambda: DeepOcSortOracle(**DOC_KW), seq, keep)


def test_botsort_sof_resolution_change_mid_sequence():
    """A new frame size restarts the tracker's estimator exactly as it restarts the standalone one."""
    import boxmot_b200 as bb
    from oracle.trackers import BotSortOracle
    from tests.common import assert_rows_match

    a = _seq_with_gaps(6, (360, 640), 83)
    b = _seq_with_gaps(6, (720, 1280), 84)
    gpu = bb.BotSort(cap_tracks=128, cap_dets=64, **BOT_KW)
    gpu.set_cmc("sof")
    sof, orc = bb.SOF(), BotSortOracle(**BOT_KW)
    for f, (im, d) in enumerate(a + b):
        w = sof.apply(im, d)
        assert_rows_match(gpu.update(d, im), orc.update(d, im, warp=w if _est(sof.last_status) else None), f)
        if f == 6:
            assert sof.last_status == 0


def test_multistream_sof_matches_standalone_per_stream():
    """8 streams in one tracker: every stream's rows are bit-identical to a single-stream tracker fed the standalone
    estimator's warps for that stream's sequence (so each stream's estimate is the standalone one, bit for bit)."""
    import boxmot_b200 as bb

    S, n = 8, 10
    seqs = [_seq_with_gaps(n, (360, 640), 90 + s) for s in range(S)]
    multi = bb.MultiStreamTracker("botsort", n_streams=S, cap_tracks=128, cap_dets=64, feat_dim=512, **BOT_KW)
    multi.set_cmc("sof")
    singles = [bb.BotSort(cap_tracks=128, cap_dets=64, **BOT_KW) for _ in range(S)]
    sofs = [bb.SOF() for _ in range(S)]
    estimated = 0
    for f in range(n):
        got = multi.update([seqs[s][f][1] for s in range(S)], [seqs[s][f][0] for s in range(S)])
        for s in range(S):
            im, d = seqs[s][f]
            w = sofs[s].apply(im, d)
            estimated += _est(sofs[s].last_status)
            want = singles[s].update(d, im, warp=w if _est(sofs[s].last_status) else None)
            np.testing.assert_array_equal(np.asarray(got[s]), np.asarray(want), err_msg=f"stream {s} frame {f}")
    assert estimated >= S * (n - 3)


def test_tracker_set_cmc_abi():
    import boxmot_b200 as bb

    for kind, ok in (("botsort", True), ("deepocsort", True), ("strongsort", False), ("bytetrack", False)):
        t = bb.MultiStreamTracker(kind, n_streams=1, cap_tracks=64, cap_dets=32, feat_dim=512)
        assert bool(t.lib.boxmot_b200_tracker_set_cmc(t.handle, b"sof")) == ok, kind
        assert t.lib.boxmot_b200_tracker_set_cmc(t.handle, None) == 1
        t.close()
