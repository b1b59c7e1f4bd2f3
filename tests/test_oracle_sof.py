"""The SOF camera-motion estimator without a GPU: tests/sof_oracle.py against the golden of the unmodified reference
class, and the host build of boxmot_b200/csrc/cmc_sof.cuh (tests/sofsim.py) stage by stage against the installed OpenCV
and as a whole against the oracle.  The GPU tests then pin the kernels on the same host build bit for bit."""
from pathlib import Path

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from boxmot_b200.synthetic import camera_pan_sequence, camera_similarity_sequence  # noqa: E402
from tests import sofsim  # noqa: E402
from tests.sof_oracle import CORNERS, LK, SUBPIX_CRIT, SofOracle, corner_mask, preprocess  # noqa: E402

GOLDEN = np.load(Path(__file__).parent / "golden" / "cmc_sof.npz")
SEQS = {"sim360": ("sim", (360, 640), 21), "sim720": ("sim", (720, 1280), 22), "pan360": ("pan", (360, 640), 23)}


def _seq(kind, hw, seed, n=8):
    if kind == "sim":
        f, d, _ = camera_similarity_sequence(n, hw=hw, seed=seed)
    else:
        f, d, _, _ = camera_pan_sequence(n, hw=hw, seed=seed)
    return f, d


def _gray_pairs():
    """(prev, cur) registration images: synthetic similarity motion at three sizes and consecutive MOT17 frames."""
    out = []
    for hw, seed in (((360, 640), 31), ((720, 1280), 32), ((1080, 1920), 33), ((475, 801), 34)):
        f, _ = _seq("sim", hw, seed, n=2)
        out.append((preprocess(f[0]), preprocess(f[1])))
    reg = GOLDEN["mot17_reg"]
    out += [(reg[i], reg[i + 1]) for i in (0, 1, 5, 6)]
    return out


def _is_eye(w):
    return np.array_equal(w, np.eye(2, 3, dtype=np.float32))


@pytest.mark.parametrize("name", sorted(SEQS))
def test_oracle_matches_reference_golden(name):
    frames, dets = _seq(*SEQS[name])
    ref = GOLDEN[f"{name}_warps"]
    orc = SofOracle()
    got = np.stack([orc.apply(f, d) for f, d in zip(frames, dets)])
    assert [_is_eye(w) for w in got] == [_is_eye(w) for w in ref]
    assert sum(not _is_eye(w) for w in ref) >= 5
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-5)


def test_oracle_matches_reference_golden_on_mot17():
    """The reference's warps on MOT17-mini frames (two sequences of 4 and 5 frames): the oracle at scale 1 on the stored
    registration images (gray -> BGR -> gray is exact) gives the same warps, translation / 0.15 in float32."""
    reg, ref = GOLDEN["mot17_reg"], GOLDEN["mot17_warps"]
    for seq in (range(0, 4), range(4, 9)):
        orc = SofOracle(scale=1.0)
        for i in seq:
            w = orc.apply(cv2.cvtColor(reg[i], cv2.COLOR_GRAY2BGR))
            w[:, 2] = w[:, 2] / np.float32(0.15)
            assert _is_eye(w) == _is_eye(ref[i]), i
            np.testing.assert_allclose(w, ref[i], rtol=0, atol=1e-5)
    assert sum(not _is_eye(w) for w in ref) >= 5


def test_mask_matches_generate_mask():
    rng = np.random.default_rng(3)
    for h, w in ((54, 96), (108, 192), (162, 288), (71, 120)):
        d = rng.uniform(-100, 2100, (40, 4)).astype(np.float32)
        d[:, 2:] = d[:, :2] + rng.uniform(-50, 400, (40, 2)).astype(np.float32)
        d[0] = [0.0, 0.0, 1e5, 1e5]   # covers everything once clamped
        d[1] = [-3.9, -7.0, 6.67, 6.67]   # truncation toward zero on both sides
        gray = np.zeros((h, w), np.uint8)
        for k in (0, 1, 2, 40):
            sub = d[2 - min(k, 2):][:k] if k else None
            np.testing.assert_array_equal(sofsim.mask(h, w, sub), corner_mask(gray, sub))


@pytest.mark.parametrize("i", range(8))
def test_eigenvalue_map_and_corners_match_opencv(i):
    g = _gray_pairs()[i][0]
    want = cv2.cornerMinEigenVal(g, 3, 3)
    got = sofsim.eig(g)
    rel = np.abs(got - want).max() / np.abs(want).max()
    m = corner_mask(g, None)
    k = cv2.goodFeaturesToTrack(g, mask=m, **CORNERS).reshape(-1, 2)
    c = sofsim.corners(g, m)
    common = len(set(map(tuple, k)) & set(map(tuple, c)))
    same = len(k) == len(c) and bool(np.array_equal(k, c))
    print(f"eig rel {rel:.2e}, corners {len(c)} vs cv2 {len(k)}, in common {common}, identical list {same}")
    assert rel < 1e-6
    assert common >= 0.99 * len(k) and abs(len(c) - len(k)) <= 0.01 * len(k)


@pytest.mark.parametrize("i", range(8))
def test_subpix_and_lk_match_opencv(i):
    prev, cur = _gray_pairs()[i]
    k = cv2.goodFeaturesToTrack(prev, mask=corner_mask(prev, None), **CORNERS)
    sp = sofsim.subpix(prev, k.reshape(-1, 2))
    cv2.cornerSubPix(prev, k, (5, 5), (-1, -1), SUBPIX_CRIT)
    d = np.abs(sp - k.reshape(-1, 2)).max(1)
    # OpenCV's getRectSubPix uses the same replicated border, but forms its samples in another float order (measured
    # on these images: up to 3e-5 gray levels from the plain bilinear sum used here, inside and at the edges).  Where
    # the 13x13 window crosses the image edge the replicated rows make the 2x2 system nearly singular, and a point
    # there can converge to another end point (observed: corners within 7 px of the top edge only, 0-3 per image).
    # Points whose window stays inside agree within 1e-3 px.
    xy = k.reshape(-1, 2)
    inside = (xy[:, 0] >= 7) & (xy[:, 0] <= prev.shape[1] - 8) & (xy[:, 1] >= 7) & (xy[:, 1] <= prev.shape[0] - 8)
    print(f"cornerSubPix: {int((d > 1e-3).sum())} of {len(d)} beyond 1e-3 px ({int((d[inside] > 1e-3).sum())} inside)")
    assert d[inside].max() <= 1e-3 and np.mean(d <= 1e-3) >= 0.95
    assert sofsim.levels(*prev.shape) == len(cv2.buildOpticalFlowPyramid(prev, (21, 21), 3, withDerivatives=False)[1])
    nxt, st, _ = cv2.calcOpticalFlowPyrLK(prev, cur, k, None, **LK)
    n2, s2 = sofsim.lk(prev, cur, k.reshape(-1, 2))
    st, nxt = st.reshape(-1), nxt.reshape(-1, 2)
    both = (st == 1) & (s2 == 1)
    err = np.abs(n2[both] - nxt[both]).max()
    print(f"LK: status equal {np.mean(st == s2):.4f}, valid {int(both.sum())}/{len(st)}, max position error {err:.2e}")
    assert np.mean(st == s2) >= 0.995 and both.sum() >= 0.5 * len(st)
    assert err < 1e-3


@pytest.mark.parametrize("i", range(8))
def test_ransac_and_refine_match_opencv(i):
    prev, cur = _gray_pairs()[i]
    k = cv2.goodFeaturesToTrack(prev, mask=corner_mask(prev, None), **CORNERS)
    nxt, st, _ = cv2.calcOpticalFlowPyrLK(prev, cur, k, None, **LK)
    pv, nv = k[st.reshape(-1) == 1].reshape(-1, 2), nxt[st.reshape(-1) == 1].reshape(-1, 2)
    rng = np.random.default_rng(i)
    nv = nv.copy()
    out = rng.random(len(nv)) < 0.3   # outliers, so RANSAC has something to reject
    nv[out] += rng.uniform(-20, 20, (int(out.sum()), 2)).astype(np.float32)
    H, inl = cv2.estimateAffinePartial2D(pv, nv, method=cv2.RANSAC, ransacReprojThreshold=3.0)
    M, inl2 = sofsim.ransac(pv, nv)
    np.testing.assert_array_equal(inl.reshape(-1), inl2)
    np.testing.assert_allclose(M[:, :2], H[:, :2], rtol=0, atol=1e-6)
    np.testing.assert_allclose(M[:, 2], H[:, 2], rtol=0, atol=1e-5)


def test_two_point_model_matches_opencv():
    rng = np.random.default_rng(7)
    for _ in range(20):
        s = rng.uniform(0, 300, (2, 2)).astype(np.float32)
        d = (s * rng.uniform(0.9, 1.1) + rng.uniform(-9, 9, 2)).astype(np.float32)
        H, _ = cv2.estimateAffinePartial2D(s, d, method=cv2.RANSAC)
        M, _ = sofsim.ransac(s, d)
        np.testing.assert_allclose(M, H, rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize("hw,seed", [((360, 640), 41), ((720, 1280), 42), ((1080, 1920), 43), ((475, 801), 44)])
def test_host_sof_matches_oracle(hw, seed):
    frames, dets = _seq("sim", hw, seed, n=6)
    host, orc = sofsim.HostSOF(), SofOracle()
    for f, (im, d) in enumerate(zip(frames, dets)):
        got, want = host.apply(im, d), orc.apply(im, d)
        assert host.status == orc.status, f
        np.testing.assert_allclose(got[:, :2], want[:, :2], rtol=0, atol=1e-4)
        np.testing.assert_allclose(got[:, 2], want[:, 2], rtol=0, atol=0.02)
    assert orc.status == 1


@pytest.mark.parametrize("kind", ["constant", "covered", "inverted", "few_inliers"])
def test_failure_paths_match_oracle(kind):
    frames, dets = _seq("sim", (360, 640), 51, n=4)
    kw = dict(min_inliers=5000) if kind == "few_inliers" else {}
    host, orc = sofsim.HostSOF(**kw), SofOracle(**kw)
    seq = [(f, d) for f, d in zip(frames, dets)]
    if kind == "constant":
        seq.insert(2, (np.full_like(frames[0], 128), dets[0]))
    elif kind == "covered":
        seq.insert(1, (frames[1], np.array([[-10, -10, 700, 400]], np.float32)))
    elif kind == "inverted":
        seq.insert(2, (255 - frames[1], dets[1]))
    statuses = []
    for im, d in seq:
        got, want = host.apply(im, d), orc.apply(im, d)
        assert host.status == orc.status
        statuses.append(orc.status)
        np.testing.assert_allclose(got[:, :2], want[:, :2], rtol=0, atol=1e-4)
        np.testing.assert_allclose(got[:, 2], want[:, 2], rtol=0, atol=0.02)
    print(kind, statuses)
    assert 2 in statuses or kind == "covered"
    if kind == "few_inliers":
        assert 1 not in statuses
