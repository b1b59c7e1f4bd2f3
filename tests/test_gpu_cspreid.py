"""CSPReID-n on the GPU: each new kernel on its own against float64 (the SILU and SILU_RES tensor-core convolutions at
every shape the model runs, with slice-pitch inputs, residuals and outputs and M tails straddling crops; the stem; the
SPPF pools at the borders and at odd sizes; the attention; the head's pools and interleave), every debug tap against
the float64 oracle (tests/cspreid_oracle.py), embeddings against the oracle at 1, chunk - 1, chunk and chunk + 1 crops
in both preprocess modes at both crop sizes and against the reference golden, the five appearance trackers with
on-device CSPReID-n against the oracle trackers, the pipelined path, create_tracker with a cspreid_n_market1501.pt
checkpoint and the reference ABI.  Embedding bound as for every other backbone: max |delta| <= 1e-4 * ||e||_inf per
row, cosine > 0.999999."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tests import cspreid_oracle as oc
from tests import vit_oracle as ov
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match

CHUNK = 256


class _DeviceOracle:
    """The float64 oracle evaluated by PyTorch on the GPU on crops staged by the oracle's CPU restatement."""

    def __init__(self, sd, hw=(256, 128), preprocess="resize"):
        self.sd = {k: v.cuda() for k, v in oc.double_state(sd).items()}
        self.hw = hw
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        x = ov.get_crops(xyxys, img, self.preprocess, self.hw)
        f = torch.cat([oc.embed(self.sd, x[i:i + 64].cuda().double()) for i in range(0, len(x), 64)])
        return f.cpu().numpy().astype(np.float32)


def _state(seed):
    from boxmot_b200.synthetic import make_cspreid_state

    return make_cspreid_state(seed)


def _model(tmp_path, sd, fname="cspreid_n_market1501.pt", **kw):
    from boxmot_b200.reid import B200ReID

    pt = tmp_path / fname
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    return B200ReID(pt, **kw)


def _emb_ok(got, want):
    assert got.shape == want.shape
    err = np.abs(got - want).max(axis=1)
    bound = 1e-4 * np.abs(want).max(axis=1)
    assert (err <= bound).all(), f"embedding error {err.max():.3e} exceeds 1e-4*||e||inf ({bound.min():.3e})"
    assert (got.astype(np.float64) * want).sum(1).min() > 0.999999


def _boxes(rng, n, h, w):
    cx, cy = rng.uniform(0, w, n), rng.uniform(0, h, n)
    bw, bh = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    return np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)


# (crops, h, w, c0, in_ld, in_off, k, stride, N, residual, out_ld, out_off): every conv shape of the model at 256x128
# (and a few at 256x256), the bottlenecks reading / writing their C3k2 slices; 2-3 crops of 8x4 .. 64x32 maps make the
# 128-row M tiles straddle crops, and the off-grid sizes leave M tails.
CONV_CASES = [
    (3, 64, 32, 32, 32, 0, 3, 2, 64, False, 64, 0),        # stem.1
    (2, 32, 16, 64, 64, 0, 1, 1, 128, False, 192, 0),      # stage1 cv1 into its concatenation
    (2, 32, 16, 64, 192, 64, 1, 1, 32, False, 32, 0),      # stage1 bottleneck cv1 from slice 1
    (2, 32, 16, 32, 32, 0, 3, 1, 64, True, 192, 128),      # stage1 bottleneck cv2 + shortcut into slice 2
    (2, 32, 16, 192, 192, 0, 1, 1, 128, False, 128, 0),    # stage1 cv2
    (3, 32, 16, 128, 128, 0, 3, 2, 128, False, 128, 0),    # stage1 downsample
    (3, 16, 8, 128, 384, 128, 1, 1, 64, False, 64, 0),     # stage2 bottleneck cv1
    (3, 16, 8, 64, 64, 0, 3, 1, 128, True, 384, 256),      # stage2 bottleneck cv2
    (3, 16, 8, 256, 256, 0, 3, 2, 256, False, 256, 0),     # stage2 downsample
    (3, 8, 4, 256, 256, 0, 1, 1, 384, False, 768, 0),      # stage3 cv1
    (3, 8, 4, 192, 768, 384, 1, 1, 96, False, 96, 0),      # stage3 second bottleneck cv1 (N 96: BN 32 tiles)
    (3, 8, 4, 96, 96, 0, 3, 1, 192, True, 768, 576),       # stage3 second bottleneck cv2 (N 192: BN 64 tiles)
    (3, 8, 4, 384, 384, 0, 3, 2, 384, False, 384, 0),      # stage3 downsample
    (5, 8, 4, 384, 384, 0, 1, 1, 512, False, 768, 0),      # stage4 cv1
    (5, 8, 4, 128, 128, 0, 3, 1, 256, True, 768, 512),     # stage4 bottleneck cv2
    (5, 8, 4, 512, 512, 0, 1, 1, 256, False, 1024, 0),     # SPPF cv1
    (5, 8, 8, 1024, 1024, 0, 1, 1, 512, False, 512, 0),    # SPPF cv2 at 256x256
    (2, 7, 5, 96, 96, 0, 3, 1, 192, True, 768, 576),       # odd map: M tail, 35-row crops
    (3, 9, 5, 64, 192, 64, 3, 2, 32, False, 32, 0),        # odd map, stride 2, pitched 3x3 input
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n{}_{}x{}_c{}ld{}+{}_k{}s{}_N{}{}_ld{}+{}".format(
    *c[:9], "_res" if c[9] else "", c[10], c[11]))
def test_cspreid_conv_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h, w, c0, in_ld, in_off, k, s, N, with_res, out_ld, out_off = case
    rng = np.random.default_rng(abs(hash(case)) & 0xffff)
    Ho, Wo = (h - 1) // s + 1, (w - 1) // s + 1
    x = rng.standard_normal((n, h, w, in_ld)).astype(np.float32)
    wt = (rng.standard_normal((k * k * c0, N)) / np.sqrt(k * k * c0)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    res = rng.standard_normal((n, Ho, Wo, out_ld)).astype(np.float32) if with_res else None
    out = np.full((n, Ho, Wo, out_ld), np.nan, np.float32)
    for off, count in ((0, n + 3), (1, n)):   # every crop (the count clamps to the arrays), then all but the last
        o = out.copy()
        k_ = min(count - off, n)
        ok = lib.boxmot_b200_cspreid_conv(x.ctypes.data, n, off, count, h, w, c0, in_ld, in_off, k, s, wt.ctypes.data, N,
                                          b.ctypes.data, res.ctypes.data if with_res else None, out_ld, out_off,
                                          o.ctypes.data, out_ld, out_off)
        assert ok, _lib.last_error(lib)
        xs = torch.from_numpy(x[..., in_off:in_off + c0]).double().permute(0, 3, 1, 2)
        wk = torch.from_numpy(wt).double().reshape(k, k, c0, N).permute(3, 2, 0, 1)
        acc = F.conv2d(xs, wk, torch.from_numpy(b).double(), s, k // 2)
        mag = F.conv2d(xs.abs(), wk.abs(), torch.from_numpy(b).double().abs(), s, k // 2).permute(0, 2, 3, 1).numpy()
        want = F.silu(acc).permute(0, 2, 3, 1).numpy()
        if with_res:
            want = want + res[..., out_off:out_off + N]
        got = o[..., out_off:out_off + N]
        err = np.abs(got[:k_] - want[:k_])
        assert (err <= 1e-5 * (mag[:k_] + 1.0)).all(), f"max err {np.nanmax(err):.3e}"
        assert np.isnan(got[k_:]).all(), "a crop outside the window was written"
        rest = np.delete(o, np.s_[out_off:out_off + N], axis=3)
        assert np.isnan(rest).all(), "columns outside the slice were written"


@pytest.mark.parametrize("hw", [(256, 128), (256, 256), (31, 17)])
def test_cspreid_stem_matches_float64(hw):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(hw[1])
    n, (h, w) = 3, hw
    x = rng.standard_normal((n, h, w, 3)).astype(np.float32)
    wt = (rng.standard_normal((27, 32)) / 5).astype(np.float32)
    b = rng.standard_normal(32).astype(np.float32)
    Ho, Wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out = np.full((n, Ho, Wo, 32), np.nan, np.float32)
    assert lib.boxmot_b200_cspreid_map(0, x.ctypes.data, n, 1, n, h, w, 3, wt.ctypes.data, b.ctypes.data,
                                       out.ctypes.data), _lib.last_error(lib)
    wk = torch.from_numpy(wt).double().reshape(3, 3, 3, 32).permute(3, 2, 0, 1)
    want = F.silu(F.conv2d(torch.from_numpy(x).double().permute(0, 3, 1, 2), wk, torch.from_numpy(b).double(), 2, 1))
    want = want.permute(0, 2, 3, 1).numpy()
    assert np.isnan(out[-1]).all()
    assert np.abs(out[:-1] - want[:-1]).max() < 1e-5 * (1 + np.abs(want).max())


@pytest.mark.parametrize("hw", [(8, 4), (8, 8), (1, 1), (2, 3), (7, 5), (13, 9)])
def test_cspreid_sppf_pools_match_float64(hw):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, c, (h, w) = 3, 256, hw
    rng = np.random.default_rng(h * 31 + w)
    buf = np.full((n, h, w, 4 * c), np.nan, np.float32)
    buf[..., :c] = rng.standard_normal((n, h, w, c))
    out = buf.copy()
    assert lib.boxmot_b200_cspreid_map(1, buf.ctypes.data, n, 1, n, h, w, c, None, None, out.ctypes.data), \
        _lib.last_error(lib)
    x = torch.from_numpy(buf[..., :c]).permute(0, 3, 1, 2)
    y1 = F.max_pool2d(x, 3, 1, 1)
    y2 = F.max_pool2d(y1, 3, 1, 1)
    want = torch.cat([x, y1, y2, F.max_pool2d(y2, 3, 1, 1)], 1).permute(0, 2, 3, 1).numpy()
    assert np.array_equal(out[:-1], want[:-1]), "max pools are exact"
    assert np.array_equal(out[-1, ..., :c], buf[-1, ..., :c]) and np.isnan(out[-1, ..., c:]).all()


def _attn_params(rng):
    return [(rng.standard_normal((512, 64)) / 20).astype(np.float32), (rng.standard_normal((64, 512)) / 6).astype(np.float32),
            (rng.standard_normal((9, 512)) / 3).astype(np.float32), rng.standard_normal(512).astype(np.float32),
            (rng.standard_normal(512) / 20).astype(np.float32)]


@pytest.mark.parametrize("hw", [(8, 4), (8, 8), (3, 5), (1, 1)])
def test_cspreid_attention_matches_float64(hw):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, (h, w) = 3, hw
    rng = np.random.default_rng(h * 7 + w)
    x = rng.standard_normal((n, h, w, 512)).astype(np.float32)
    w1, w2, dw, db, ws = _attn_params(rng)
    params = np.concatenate([a.ravel() for a in (w1, w2, dw, db, ws)])
    out = np.full_like(x, np.nan)
    assert lib.boxmot_b200_cspreid_attention(x.ctypes.data, n, 1, n, h, w, params.ctypes.data, out.ctypes.data), \
        _lib.last_error(lib)
    t = lambda a: torch.from_numpy(a).double()   # noqa: E731
    xx = t(x).permute(0, 3, 1, 2)
    ca = torch.sigmoid(F.silu(xx.mean((2, 3)) @ t(w1)) @ t(w2))[:, :, None, None]
    g = xx * ca
    d = F.silu(F.conv2d(g, t(dw).T.reshape(512, 1, 3, 3), t(db), 1, 1, 1, 512))
    want = (g * torch.sigmoid((d * t(ws)[None, :, None, None]).sum(1, keepdim=True))).permute(0, 2, 3, 1).numpy()
    assert np.isnan(out[-1]).all()
    assert np.abs(out[:-1] - want[:-1]).max() < 2e-5 * (1 + np.abs(want).max())


@pytest.mark.parametrize("hw", [(8, 4), (8, 8), (5, 3), (2, 1)])
def test_cspreid_head_interleave_matches_float64(hw):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, (h, w) = 7, hw
    rng = np.random.default_rng(h + 11 * w)
    x = rng.standard_normal((n, h, w, 512)).astype(np.float32)
    ws = [((rng.standard_normal((512, 512)) / 22).astype(np.float32), rng.standard_normal(512).astype(np.float32))
          for _ in range(3)]
    params = np.concatenate([a.ravel() for wb in ws for a in wb])
    rows = np.array([9, 3, 0, 5, 1, 7, 2], np.int32)
    out = np.full((10, 1536), np.nan, np.float32)
    raw = np.full((n, 1536), np.nan, np.float32)
    off = 1
    assert lib.boxmot_b200_cspreid_head(x[off:].ctypes.data, n - off, off, n, h, w, params.ctypes.data,
                                        rows.ctypes.data, 10, out.ctypes.data, raw.ctypes.data), _lib.last_error(lib)
    xx = torch.from_numpy(x[off:]).double().permute(0, 3, 1, 2)
    pools = [xx.mean((2, 3)), *F.adaptive_avg_pool2d(xx, (2, 1))[:, :, :, 0].unbind(2)]
    want = torch.stack([p @ torch.from_numpy(W).double() + torch.from_numpy(b).double()
                        for p, (W, b) in zip(pools, ws)], 2).flatten(1).numpy()
    assert np.abs(raw[: n - off] - want).max() < 1e-5 * (1 + np.abs(want).max())
    assert np.isnan(raw[n - off:]).all()
    e = want / np.linalg.norm(want, axis=1, keepdims=True)
    got = out[rows[off:]]
    assert np.abs(got - e).max() < 1e-5
    untouched = np.setdiff1d(np.arange(10), rows[off:])
    assert np.isnan(out[untouched]).all()


@pytest.mark.parametrize("fname,hw", [("cspreid_n_market1501.pt", (256, 128)), ("cspreid_n_veri.pt", (256, 256))])
def test_cspreid_every_stage_matches_oracle(tmp_path, fname, hw):
    sd = _state(11)
    reid = _model(tmp_path, sd, fname)
    assert reid.input_shape == hw and reid.feature_dim == 1536
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    x = ov.get_crops(boxes, img, "resize", hw)
    want = oc.forward_taps({k: v.cuda() for k, v in oc.double_state(sd).items()}, x.cuda().double())
    crops = reid.debug_stage(boxes, img, 0).reshape(-1, *hw, 3)
    assert np.array_equal(crops, x.permute(0, 2, 3, 1).numpy()), "crop staging must be bit-exact"
    for idx in range(1, oc.TAPS):
        w = oc.nhwc(want[idx]).cpu().numpy()
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (idx, g.shape, w.shape)
        err = np.abs(g - w).max()
        print(f"tap {idx}: max err {err:.3e} of {np.abs(w).max():.3e}")
        # tf32x3 products keep ~2^-21 of each term; over 25 layers with maps up to ~100 the maps drift to ~1.3e-4
        # of their peak (PyTorch's float32 CPU forward: ~3e-6), the same bound as the ViT taps
        assert err < 5e-4 * max(1.0, float(np.abs(w).max())), f"stage {idx}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("key", ["cspreid_n_market1501", "cspreid_n_veri"])
def test_cspreid_matches_reference_golden(tmp_path, key, mode):
    from boxmot_b200.synthetic import make_cspreid_state

    z = np.load(GOLDEN / "reid_cspreid_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    sd = make_cspreid_state(int(z[f"{key}_seed"]), num_classes=int(z["num_classes"]))
    reid = _model(tmp_path, sd, key + ".pt", preprocess=mode)
    hw = tuple(int(v) for v in z[f"{key}_input_hw"])
    assert reid.input_shape == hw
    crops = reid.debug_stage(z["boxes"], img, 0).reshape(-1, *hw, 3).transpose(0, 3, 1, 2)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"{key}_crops_sha256_{mode}"])
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"{key}_features_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("fname,hw", [("cspreid_n_market1501.pt", (256, 128)), ("cspreid_n_veri.pt", (256, 256))])
@pytest.mark.parametrize("n", [1, CHUNK - 1, CHUNK, CHUNK + 1])
def test_cspreid_batch_embeddings_match_oracle(tmp_path, n, fname, hw, mode):
    sd = _state(2)
    reid = _model(tmp_path, sd, fname, preprocess=mode)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd, hw, mode).get_features(boxes, img))
    # a crop's row does not depend on its chunk or on its position in it
    tail = slice(max(0, n - 5), n)
    assert np.array_equal(reid.get_features(boxes[tail], img), got[tail])


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort", "boosttrack", "occluboost"])
def test_cspreid_trackers_match_oracle(tmp_path, kind):
    import boxmot_b200 as bb
    from oracle.streams import bench_stream

    sd = _state(5)
    reid = _model(tmp_path, sd)
    oracle_reid = _DeviceOracle(sd)
    img, frames = bench_stream(32, 12, hw=(360, 640))
    if kind == "botsort":
        from oracle.trackers import BotSortOracle

        orc = BotSortOracle(reid_model=oracle_reid, **BOTSORT_YAML)
        gpu = bb.BotSort(reid_model=reid, cap_tracks=128, cap_dets=64, **BOTSORT_YAML)
    elif kind == "deepocsort":
        from oracle.deepocsort import DeepOcSortOracle

        orc = DeepOcSortOracle(reid_model=oracle_reid)
        gpu = bb.DeepOcSort(reid_model=reid, cap_tracks=128, cap_dets=64)
    elif kind == "strongsort":
        from oracle.strongsort import StrongSortOracle

        kw = dict(min_conf=0.3, max_cos_dist=0.4, n_init=2)
        orc = StrongSortOracle(reid_model=oracle_reid, **kw)
        gpu = bb.StrongSort(reid_model=reid, cap_tracks=128, cap_dets=64, **kw)
    elif kind == "boosttrack":
        from tests.boosttrack_oracle import BoostTrackOracle

        kw = dict(det_thresh=0.5, use_rich_s=True, use_sb=True, use_vt=True, with_reid=True)
        orc = BoostTrackOracle(reid_model=oracle_reid, **kw)
        gpu = bb.BoostTrack(reid_model=reid, use_cmc=False, cap_tracks=128, cap_dets=64, **kw)
    else:
        from tests.occluboost_oracle import OccluBoostOracle

        kw = dict(det_thresh=0.5, with_reid=True, use_second_pass=True)
        orc = OccluBoostOracle(reid_model=oracle_reid, **kw)
        gpu = bb.OccluBoost(reid_model=reid, use_cmc=False, cap_tracks=128, cap_dets=64, **kw)
    n_rows = 0
    for f, d in enumerate(frames):
        got = gpu.update(d, img)
        want = np.asarray(orc.update(d, img), np.float32).reshape(-1, np.asarray(got).shape[1])
        assert_rows_match(got, want, f)
        n_rows += len(got)
    assert n_rows > 0


def test_cspreid_pipelined_device_path_equals_synchronous(tmp_path):
    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state(3), tmp_path / "pipe.b200reid")
    img, dets = bench_stream(48, 16, hw=(360, 640))
    imgs = np.stack([np.roll(img, 7 * k, axis=1) for k in range(4)])
    d_imgs = torch.from_numpy(imgs).cuda()
    d_dets = torch.from_numpy(np.stack(dets)[:, None].astype(np.float32)).cuda().contiguous()
    rows = (ctypes.c_int * 1)(48)
    snaps = []
    kw = dict(track_high_thresh=0.6, new_track_thresh=0.62, appearance_thresh=0.6, proximity_thresh=0.6)
    for sync in (1, 0):
        trk = bb.MultiStreamTracker("botsort", n_streams=1, cap_tracks=256, cap_dets=48, feat_dim=1536,
                                    reid_blob=str(blob), **kw)
        for f in range(len(dets)):
            ok = lib.boxmot_b200_tracker_update_device(trk.handle, d_dets[f].data_ptr(), rows, None,
                                                       d_imgs[f % 4].data_ptr(), 360, 640, sync)
            assert ok, _lib.last_error(lib)
        out = np.zeros((48, 9), np.float32)
        o_ptr = (ctypes.c_void_p * 1)(out.ctypes.data)
        o_cap = (ctypes.c_int * 1)(48)
        o_rows = (ctypes.c_int * 1)()
        assert lib.boxmot_b200_tracker_fetch(trk.handle, o_ptr, o_cap, o_rows), _lib.last_error(lib)
        snaps.append((out[: o_rows[0]].copy(), trk.snapshot(0)))
        trk.close()
    (rows_a, st_a), (rows_b, st_b) = snaps
    assert rows_a.shape == rows_b.shape and len(rows_a) > 0
    assert np.array_equal(rows_a, rows_b)
    assert sorted(st_a) == sorted(st_b)
    for k in st_a:
        assert np.array_equal(st_a[k][0], st_b[k][0]) and np.array_equal(st_a[k][1], st_b[k][1])


def test_create_tracker_with_cspreid_checkpoint(tmp_path):
    """A seeded checkpoint saved as a training checkpoint (`state_dict` with `module.` prefixes, classifiers included)
    through create_tracker(reid_weights=...): converted once, 1536-d embeddings, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream

    sd = _state(4)
    pt = tmp_path / "cspreid_n_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    for kind in ("botsort", "deepocsort", "strongsort", "boosttrack", "occluboost"):
        trk = bb.create_tracker(kind, reid_weights=pt)
        img, frames = bench_stream(24, 6, hw=(360, 640))
        n = sum(len(trk.update(d, img)) for d in frames)
        assert n > 0, kind


def test_reference_abi_botsort_with_cspreid_model(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state(6), tmp_path / "abi.b200reid")
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
    dim = ctypes.c_int(0)
    assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 1536
    lib.boxmot_reid_capi_destroy(h)
    cfg = _lib.BoxMOTBotSortConfig()
    cfg.track_high_thresh, cfg.track_low_thresh, cfg.new_track_thresh = 0.6, 0.1, 0.62
    cfg.track_buffer, cfg.match_thresh, cfg.proximity_thresh, cfg.appearance_thresh = 30, 0.8, 0.6, 0.6
    cfg.cmc_method, cfg.frame_rate, cfg.fuse_first_associate, cfg.with_reid, cfg.max_obs = b"none", 30, 0, 1, 50
    cfg.reid_model_path, cfg.reid_preprocess = str(blob).encode(), b"resize"
    t = lib.boxmot_botsort_create(ctypes.byref(cfg))
    assert t, _lib.last_error(lib)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    img = np.ascontiguousarray(img)
    out = np.zeros((64, 9), np.float32)
    n_out, obb, total = ctypes.c_int(0), ctypes.c_int(0), 0
    for d in frames:
        d = np.ascontiguousarray(d, np.float32)
        ok = lib.boxmot_botsort_update(t, d.ctypes.data, len(d), 6, None, 0, 0, img.ctypes.data, 360, 640, 3,
                                       out.ctypes.data, 64, 9, ctypes.byref(n_out), ctypes.byref(obb))
        assert ok, _lib.last_error(lib)
        total += n_out.value
    lib.boxmot_botsort_destroy(t)
    assert total > 0
