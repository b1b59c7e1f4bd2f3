"""LMBN_n (lmbn_n_duke / _market / _cuhk03_d) on the GPU: 384x128 crop staging bit-exact, every stage tap against the
oracle (oracle.lmbn.lmbn_n_forward), 3584-d embeddings against the oracle and the reference-class golden at chunk
boundaries and in both preprocess modes, the three appearance trackers with on-device LMBN against the oracle
trackers, the pipelined device path, create_tracker with a .pt checkpoint and the reference ABI.
Embedding bound as for OSNet: max |delta| <= 1e-4 * ||e||_inf per row, cosine > 0.999999."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import lmbn as olm
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match

# debug_stage taps of the LMBN_n path (csrc/reid_model.cu run_lmbn_chunk) -> oracle stage names
TAPS = {1: "stem", 2: "pool", 3: "backone.2.0", 4: "backone.2.1", 5: "backone.2.2", 6: "trunk"}
for _i, _br in ((7, "global_branch"), (13, "partial_branch"), (18, "channel_branch")):
    for _j, _s in enumerate((".0.1", ".0.2", ".1.0", ".1.1", ".2")):
        TAPS[_i + _j] = _br + _s
TAPS[12] = "bottleneck"


class _DeviceOracle:
    """The oracle's LMBN_n evaluated by PyTorch on the GPU (float32, TF32 off) on crops staged by the oracle's CPU
    restatement, so that hundreds of crops finish in seconds.  Test infrastructure only."""

    def __init__(self, sd, preprocess="resize"):
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        self.sd = {k: v.cuda() for k, v in sd.items()}
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        x = olm.get_crops_hw(xyxys, img, self.preprocess, olm.LMBN_INPUT_HW).cuda()
        f = torch.cat([olm.lmbn_n_forward(self.sd, x[i:i + 64]) for i in range(0, len(x), 64)]).cpu().numpy()
        return f / np.linalg.norm(f, axis=-1, keepdims=True)


def _state(seed):
    from boxmot_b200.synthetic import make_lmbn_n_state

    return make_lmbn_n_state(seed=seed)


def _model(tmp_path, sd, name="lmbn", **kw):
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.weights import export_blob

    return B200ReID(export_blob(sd, tmp_path / f"{name}.b200reid"), **kw)


def _emb_ok(got, want):
    assert got.shape == want.shape
    err = np.abs(got - want).max(axis=1)
    bound = 1e-4 * np.abs(want).max(axis=1)
    assert (err <= bound).all(), f"embedding error {err.max():.3e} exceeds 1e-4*||e||inf ({bound.min():.3e})"
    assert (got * want).sum(1).min() > 0.999999


def _boxes(rng, n, h, w):
    cx, cy = rng.uniform(0, w, n), rng.uniform(0, h, n)
    bw, bh = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    return np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
def test_lmbn_matches_reference_golden(tmp_path, mode):
    from boxmot_b200.synthetic import make_lmbn_n_state

    z = np.load(GOLDEN / "reid_lmbn_n_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    reid = _model(tmp_path, make_lmbn_n_state(seed=int(z["weight_seed"]), num_classes=int(z["num_classes"])),
                  preprocess=mode)
    assert reid.input_shape == (384, 128) and reid.feature_dim == 3584
    crops = reid.debug_stage(z["boxes"], img, 0).reshape(-1, 384, 128, 3)
    want = olm.get_crops_hw(z["boxes"], img, mode, olm.LMBN_INPUT_HW).permute(0, 2, 3, 1).numpy()
    assert np.array_equal(crops, want), "crop staging must be bit-exact"
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"features_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


def test_lmbn_every_stage_matches_oracle(tmp_path):
    sd = _state(11)
    reid = _model(tmp_path, sd)
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    _, want = olm.lmbn_n_forward(sd, olm.get_crops_hw(boxes, img, "resize", olm.LMBN_INPUT_HW), return_stages=True)
    for idx, name in TAPS.items():
        w = want[name].permute(0, 2, 3, 1).contiguous().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        err = np.abs(g - w).max()
        assert err < 2e-5 * max(1.0, float(np.abs(w).max())), f"stage {idx} {name}: max err {err:.3e}"


@pytest.mark.parametrize("n", [1, 7, 131, 256])
def test_lmbn_batch_embeddings_match_oracle(tmp_path, n):
    sd = _state(2)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd).get_features(boxes, img))
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    assert reid.get_features(np.zeros((0, 4), np.float32), img).size == 0


def test_lmbn_resize_pad_and_tensor_core_switch(tmp_path, monkeypatch):
    """resize_pad staging through the whole network, and BOXMOT_B200_REID_TC=1 (the opt-in tensor-core pointwise GEMM of
    the OSNet path) leaves LMBN_n on its float32 kernels: identical rows."""
    sd = _state(13)
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.concatenate([_boxes(rng, 40, 480, 640), [[5, 5, 300, 470], [-30, -30, -5, -5], [600, 400, 800, 700]]])
    boxes = boxes.astype(np.float32)
    pad = _model(tmp_path, sd, "pad", preprocess="resize_pad")
    _emb_ok(pad.get_features(boxes, img), _DeviceOracle(sd, "resize_pad").get_features(boxes, img))
    base = _model(tmp_path, sd, "base").get_features(boxes, img)
    monkeypatch.setenv("BOXMOT_B200_REID_TC", "1")
    assert np.array_equal(_model(tmp_path, sd, "tc").get_features(boxes, img), base)


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_lmbn_trackers_match_oracle(tmp_path, kind):
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
    else:
        from oracle.strongsort import StrongSortOracle

        kw = dict(min_conf=0.3, max_cos_dist=0.4, n_init=2)
        orc = StrongSortOracle(reid_model=oracle_reid, **kw)
        gpu = bb.StrongSort(reid_model=reid, cap_tracks=128, cap_dets=64, **kw)
    n_rows = 0
    for f, d in enumerate(frames):
        got = gpu.update(d, img)
        assert_rows_match(got, orc.update(d, img), f)
        n_rows += len(got)
    assert n_rows > 0


def test_lmbn_pipelined_device_path_equals_synchronous(tmp_path):
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
        trk = bb.MultiStreamTracker("botsort", n_streams=1, cap_tracks=256, cap_dets=48, feat_dim=3584,
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


def test_create_tracker_with_lmbn_checkpoint(tmp_path):
    """A seeded checkpoint saved like the released lmbn_n_duke.pt (`state_dict` with `module.` prefixes) through
    create_tracker("botsort", reid_weights=...): converted once, 3584-d embeddings on the device, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream

    sd = _state(4)
    pt = tmp_path / "lmbn_n_duke.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    n = sum(len(trk.update(d, img)) for d in frames)
    assert n > 0


def test_reference_abi_botsort_with_lmbn_model(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state(6), tmp_path / "abi.b200reid")
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
    dim = ctypes.c_int(0)
    assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 3584
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
    out = np.zeros((64, 9), np.float32)   # the reference ABI's track rows have 9 columns
    n_out, obb, total = ctypes.c_int(0), ctypes.c_int(0), 0
    for d in frames:
        d = np.ascontiguousarray(d, np.float32)
        ok = lib.boxmot_botsort_update(t, d.ctypes.data, len(d), 6, None, 0, 0, img.ctypes.data, 360, 640, 3,
                                       out.ctypes.data, 64, 9, ctypes.byref(n_out), ctypes.byref(obb))
        assert ok, _lib.last_error(lib)
        total += n_out.value
    lib.boxmot_botsort_destroy(t)
    assert total > 0
