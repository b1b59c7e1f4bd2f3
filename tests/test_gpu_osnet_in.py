"""OSNet-AIN (osnet_ain_x1_0 / _x0_75 / _x0_5 / _x0_25) and OSNet-IBN (osnet_ibn_x1_0) on the GPU: the instance-norm
kernels against float64, every stage tap against the oracle (oracle.osnet_in), 512-d embeddings against the reference
golden and the oracle across the chunk boundary, chunk and position independence, the tensor-core switch, the three
appearance trackers with on-device OSNet-AIN against the oracle trackers, the pipelined device path, create_tracker with
a .pt checkpoint and the reference ABI.  Embedding bound as for OSNet: max |delta| <= 1e-4 * ||e||_inf per row,
cosine > 0.999999."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import osnet_in as oin
from oracle.reid import get_crops
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match

# debug_stage taps (csrc/reid_model.cu, the OSNet loop) -> oracle stage names
TAPS = {1: "stem", 2: "pool", 3: "conv2.0", 4: "conv2.1", 5: "conv2.2", 6: "conv3.0", 7: "conv3.1", 8: "conv3.2",
        9: "conv4.0", 10: "conv4.1", 11: "conv5"}
BLANK = [-30, -30, -5, -5]   # entirely outside the frame: a blank crop


def _state(name, seed):
    from boxmot_b200.synthetic import make_osnet_ain_state, make_osnet_ibn_state, make_osnet_state

    if name == "osnet_ibn_x1_0":
        return make_osnet_ibn_state(seed=seed)
    if name.startswith("osnet_ain"):
        return make_osnet_ain_state(name, seed)
    return make_osnet_state(name, seed=seed)


class _DeviceOracle:
    """The oracle's forward evaluated by PyTorch on the GPU (float32, TF32 off) on crops staged by the oracle's CPU
    restatement, so that hundreds of crops finish in seconds.  Test infrastructure only."""

    def __init__(self, sd, preprocess="resize"):
        from oracle.reid import osnet_forward

        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        self.sd = {k: v.cuda() for k, v in sd.items()}
        self.fwd = oin.osnet_in_forward if (oin.is_osnet_ain(sd) or oin.is_osnet_ibn(sd)) else osnet_forward
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        x = get_crops(xyxys, img, self.preprocess).cuda()
        f = torch.cat([self.fwd(self.sd, x[i:i + 64]) for i in range(0, len(x), 64)]).cpu().numpy()
        return f / np.linalg.norm(f, axis=-1, keepdims=True)


def _model(tmp_path, sd, name="m", **kw):
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
    b = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)
    if n > 1:
        b[n // 2] = BLANK
    return b


# ---- the kernels on their own ------------------------------------------------------------------------------------
def _in_f64(x, gamma, beta):
    x = x.astype(np.float64)
    mean = x.mean(axis=(1, 2), keepdims=True)
    var = ((x - mean) ** 2).mean(axis=(1, 2), keepdims=True)
    return (x - mean) / np.sqrt(var + 1e-5) * gamma + beta


@pytest.mark.parametrize("c", [16, 48, 64, 72, 256, 512])
def test_instance_norm_kernels_match_float64(c):
    """k_in_stats + k_in_apply with the residual added after the norm (OSNet-AIN) or none (OSNet-IBN, whose residual
    the conv3 GEMM has already added), with and without the ReLU, and the stem form fused into the 3x3 max pool.  One
    channel is constant and one nearly so."""
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(c)
    n, h, w = 3, 16, 8
    x = (rng.normal(size=(n, h, w, c)) * rng.uniform(0.1, 5, c) + rng.normal(size=c) * 3).astype(np.float32)
    x[:, :, :, 1] = 2.5
    x[:, :, :, 2] = 1.0 + (rng.normal(size=(n, h, w)) * 1e-4).astype(np.float32)
    gamma = (rng.uniform(0.5, 1.5, c) * np.where(rng.random(c) < 0.3, -1, 1)).astype(np.float32)
    beta = rng.normal(size=c).astype(np.float32)
    res = rng.normal(size=x.shape).astype(np.float32)
    ref = _in_f64(x, gamma, beta)
    for residual, relu in ((None, 0), (None, 1), (res, 1), (res, 0)):
        out = np.empty_like(x)
        ok = lib.boxmot_b200_instance_norm(x.ctypes.data, n, h, w, c, gamma.ctypes.data, beta.ctypes.data,
                                           None if residual is None else residual.ctypes.data, relu, 0, out.ctypes.data)
        assert ok, _lib.last_error(lib)
        want = ref + (0 if residual is None else residual)
        want = np.maximum(want, 0) if relu else want
        assert np.abs(out - want).max() < 4e-6 * max(1.0, np.abs(want).max()), (residual is None, relu)
    pooled = np.empty((n, h // 2, w // 2, c), np.float32)
    ok = lib.boxmot_b200_instance_norm(x.ctypes.data, n, h, w, c, gamma.ctypes.data, beta.ctypes.data, None, 1, 1,
                                       pooled.ctypes.data)
    assert ok, _lib.last_error(lib)
    want = torch.nn.functional.max_pool2d(torch.from_numpy(np.maximum(ref, 0)).permute(0, 3, 1, 2), 3, 2, 1)
    want = want.permute(0, 2, 3, 1).numpy()
    assert np.abs(pooled - want).max() < 4e-6 * max(1.0, np.abs(want).max())


# ---- the networks ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["osnet_ain_x1_0", "osnet_ain_x0_25", "osnet_ibn_x1_0"])
def test_every_stage_matches_oracle(tmp_path, name):
    sd = _state(name, 11)
    reid = _model(tmp_path, sd)
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], BLANK, [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    _, want = oin.osnet_in_forward(sd, get_crops(boxes, img), return_stages=True)
    for idx, stage in TAPS.items():
        w = want[stage].permute(0, 2, 3, 1).contiguous().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (stage, g.shape, w.shape)
        err = np.abs(g - w).max()
        assert err < 2e-5 * max(1.0, float(np.abs(w).max())), f"{name} stage {idx} {stage}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("name", ["osnet_ain_x1_0", "osnet_ain_x0_25", "osnet_ibn_x1_0"])
def test_matches_reference_golden(tmp_path, name, mode):
    from boxmot_b200.synthetic import make_osnet_ain_state, make_osnet_ibn_state

    z = np.load(GOLDEN / "reid_osnet_in_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    seed, k = int(z[f"weight_seed_{name}"]), int(z["num_classes"])
    sd = make_osnet_ibn_state(seed, num_classes=k) if "ibn" in name else make_osnet_ain_state(name, seed, num_classes=k)
    reid = _model(tmp_path, sd, preprocess=mode)
    assert reid.input_shape == (256, 128) and reid.feature_dim == 512
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"{name}_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("n", [1, 7, 131, 256, 300])
def test_batch_embeddings_match_oracle(tmp_path, n):
    sd = _state("osnet_ain_x1_0", 2)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd).get_features(boxes, img))
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    assert reid.get_features(np.zeros((0, 4), np.float32), img).size == 0


@pytest.mark.parametrize("name", ["osnet_ain_x0_75", "osnet_ain_x0_5", "osnet_ibn_x1_0", "osnet_x0_75", "osnet_x0_5"])
def test_other_widths_match_oracle(tmp_path, name):
    """x0_75 and x0_5 (mid channels 48 / 72 / 96 and 32 / 48 / 64) run the generic LightConv kernel; the plain OSNet
    widths are checked too, as no other test runs them."""
    sd = _state(name, 8)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(5)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = _boxes(rng, 40, 480, 640)
    _emb_ok(reid.get_features(boxes, img), _DeviceOracle(sd).get_features(boxes, img))


def test_chunk_and_position_independence(tmp_path):
    """The same 7 crops alone and at positions 250-256 of a 300-crop call (across the 256-crop chunk boundary) give
    bit-identical rows, for OSNet-AIN and for plain osnet_x1_0 as the control."""
    rng = np.random.default_rng(41)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    seven = _boxes(rng, 7, 720, 1280)
    many = _boxes(rng, 300, 720, 1280)
    many[250:257] = seven
    for name in ("osnet_ain_x1_0", "osnet_x1_0"):
        reid = _model(tmp_path, _state(name, 9), name)
        alone = reid.get_features(seven, img)
        inside = reid.get_features(many, img)[250:257]
        assert np.array_equal(alone, inside), name


def test_resize_pad_and_tensor_core_switch(tmp_path, monkeypatch):
    """resize_pad staging through OSNet-AIN x0_25, and BOXMOT_B200_REID_TC=1 (the opt-in tensor-core pointwise GEMM of
    the OSNet path, which also covers the x0_25 widths) leaves it on its float32 kernels: identical rows."""
    sd = _state("osnet_ain_x0_25", 13)
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.concatenate([_boxes(rng, 40, 480, 640), [[5, 5, 300, 470], [600, 400, 800, 700]]]).astype(np.float32)
    pad = _model(tmp_path, sd, "pad", preprocess="resize_pad")
    _emb_ok(pad.get_features(boxes, img), _DeviceOracle(sd, "resize_pad").get_features(boxes, img))
    base = _model(tmp_path, sd, "base").get_features(boxes, img)
    _emb_ok(base, _DeviceOracle(sd).get_features(boxes, img))
    monkeypatch.setenv("BOXMOT_B200_REID_TC", "1")
    assert np.array_equal(_model(tmp_path, sd, "tc").get_features(boxes, img), base)


# ---- trackers and loading paths ------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_trackers_match_oracle(tmp_path, kind):
    import boxmot_b200 as bb
    from oracle.streams import bench_stream

    sd = _state("osnet_ain_x1_0", 5)
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


def test_pipelined_device_path_equals_synchronous(tmp_path):
    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state("osnet_ain_x1_0", 3), tmp_path / "pipe.b200reid")
    img, dets = bench_stream(48, 16, hw=(360, 640))
    imgs = np.stack([np.roll(img, 7 * k, axis=1) for k in range(4)])
    d_imgs = torch.from_numpy(imgs).cuda()
    d_dets = torch.from_numpy(np.stack(dets)[:, None].astype(np.float32)).cuda().contiguous()
    rows = (ctypes.c_int * 1)(48)
    snaps = []
    kw = dict(track_high_thresh=0.6, new_track_thresh=0.62, appearance_thresh=0.6, proximity_thresh=0.6)
    for sync in (1, 0):
        trk = bb.MultiStreamTracker("botsort", n_streams=1, cap_tracks=256, cap_dets=48, feat_dim=512,
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


def test_create_tracker_with_ain_checkpoint(tmp_path):
    """A seeded checkpoint saved like a released osnet_ain_x1_0_msmt17.pt (`state_dict` with `module.` prefixes) through
    create_tracker("botsort", reid_weights=...): converted once, 512-d embeddings on the device, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream

    pt = tmp_path / "osnet_ain_x1_0_msmt17.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in _state("osnet_ain_x1_0", 4).items()}}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    assert sum(len(trk.update(d, img)) for d in frames) > 0


def test_reference_abi_with_ain_and_ibn_blobs(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    img, frames = bench_stream(24, 6, hw=(360, 640))
    img = np.ascontiguousarray(img)
    for name in ("osnet_ain_x1_0", "osnet_ibn_x1_0"):
        sd = _state(name, 6)
        blob = export_blob(sd, tmp_path / f"{name}.b200reid")
        h = ctypes.c_void_p()
        assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
        dim = ctypes.c_int(0)
        assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 512
        d = np.ascontiguousarray(frames[0][:, :4], np.float32)
        out = np.empty((len(d), 512), np.float32)
        assert lib.boxmot_reid_capi_compute_features(h, d.ctypes.data, len(d), img.ctypes.data, 360, 640, 3,
                                                     out.ctypes.data, out.size) == 1, _lib.last_error(lib)
        lib.boxmot_reid_capi_destroy(h)
        _emb_ok(out, _DeviceOracle(sd).get_features(d, img))
        cfg = _lib.BoxMOTBotSortConfig()
        cfg.track_high_thresh, cfg.track_low_thresh, cfg.new_track_thresh = 0.6, 0.1, 0.62
        cfg.track_buffer, cfg.match_thresh, cfg.proximity_thresh, cfg.appearance_thresh = 30, 0.8, 0.6, 0.6
        cfg.cmc_method, cfg.frame_rate, cfg.fuse_first_associate, cfg.with_reid, cfg.max_obs = b"none", 30, 0, 1, 50
        cfg.reid_model_path, cfg.reid_preprocess = str(blob).encode(), b"resize"
        t = lib.boxmot_botsort_create(ctypes.byref(cfg))
        assert t, _lib.last_error(lib)
        rows_out = np.zeros((64, 9), np.float32)
        n_out, obb, total = ctypes.c_int(0), ctypes.c_int(0), 0
        for d in frames:
            d = np.ascontiguousarray(d, np.float32)
            ok = lib.boxmot_botsort_update(t, d.ctypes.data, len(d), 6, None, 0, 0, img.ctypes.data, 360, 640, 3,
                                           rows_out.ctypes.data, 64, 9, ctypes.byref(n_out), ctypes.byref(obb))
            assert ok, _lib.last_error(lib)
            total += n_out.value
        lib.boxmot_botsort_destroy(t)
        assert total > 0
