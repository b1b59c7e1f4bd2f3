"""ResNet50 / ResNet101 on the GPU: every instance of the tensor-core convolution kernel on its own against float64,
every stage tap against the oracle (oracle.resnet.resnet_forward), 2048-d embeddings against a float64 oracle and the
reference-class golden (strict loads and a resnet50_fc512 checkpoint) at chunk boundaries and in both preprocess modes,
the three appearance trackers with on-device ResNet50 against the oracle trackers, the pipelined device path,
create_tracker with a resnet50_fc512_*.pt checkpoint and the reference ABI.
Embedding bound as for every other backbone: max |delta| <= 1e-4 * ||e||_inf per row, cosine > 0.999999."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import resnet as orn
from oracle.reid import get_crops
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match


class _DeviceOracle:
    """The oracle's ResNet evaluated by PyTorch on the GPU in float64 on crops staged by the oracle's CPU restatement.
    Test infrastructure only."""

    def __init__(self, sd, preprocess="resize"):
        self.sd = {k: v.cuda().double() for k, v in sd.items()}
        self.preprocess = preprocess

    def forward(self, x):
        return torch.cat([orn.resnet_forward(self.sd, x[i:i + 64].cuda().double()) for i in range(0, len(x), 64)])

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        f = self.forward(get_crops(xyxys, img, self.preprocess)).cpu().numpy()
        return (f / np.linalg.norm(f, axis=-1, keepdims=True)).astype(np.float32)


def _state(seed, depth=50):
    from boxmot_b200.synthetic import make_resnet_state

    return make_resnet_state(depth, seed=seed)


def _model(tmp_path, sd, name="resnet", **kw):
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.weights import export_blob

    return B200ReID(export_blob(sd, tmp_path / f"{name}.b200reid"), **kw)


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


# (crops, h0, w0, c0, k, stride, c1, N, residual): 1x1 s1 / s2, 3x3 s1 / s2 and conv3 + downsample, at both output-channel
# tiles (N = 64 and multiples of 128); layer4's 8x4 maps make 32-pixel crops, so 128-row tiles straddle crops, and the
# odd crop counts leave partial tiles
CONV_CASES = [
    (3, 64, 32, 64, 1, 1, 0, 64, False),        # layer1 conv1 (block 0)
    (3, 64, 32, 256, 1, 1, 0, 64, False),       # layer1 conv1
    (3, 64, 32, 64, 3, 1, 0, 64, False),        # layer1 conv2
    (2, 64, 32, 64, 1, 1, 0, 256, True),        # layer1 conv3 + identity
    (2, 64, 32, 64, 1, 1, 64, 256, False),      # layer1.0 conv3 + downsample (stride 1)
    (3, 64, 32, 128, 3, 2, 0, 128, False),      # layer2.0 conv2 (stride 2)
    (5, 16, 8, 256, 3, 1, 0, 256, False),       # layer3 conv2
    (5, 16, 8, 512, 1, 2, 0, 1024, False),      # a strided 1x1 alone (the downsample's own shape)
    (7, 8, 4, 512, 1, 1, 1024, 2048, False),    # layer4.0 conv3 + downsample (x from 16x8 at stride 2)
    (7, 8, 4, 2048, 1, 1, 0, 512, False),       # layer4 conv1: 32-pixel crops straddle the 128-row tiles
    (9, 8, 4, 512, 3, 1, 0, 512, False),        # layer4 conv2
    (1, 8, 4, 512, 1, 1, 0, 2048, True),        # a single crop: one partial tile
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: f"n{c[0]}_{c[1]}x{c[2]}x{c[3]}_k{c[4]}s{c[5]}_ds{c[6]}_N{c[7]}"
                                                        + ("_res" if c[8] else ""))
def test_resnet_conv_kernel_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h0, w0, c0, k, s, c1, N, with_res = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    pad = k // 2
    ho, wo = (h0 + 2 * pad - k) // s + 1, (w0 + 2 * pad - k) // s + 1
    x0 = rng.standard_normal((n, h0, w0, c0)).astype(np.float32)
    h1, w1, s1 = (2 * ho, 2 * wo, 2) if c1 >= 1024 else (ho, wo, 1)
    x1 = rng.standard_normal((n, h1, w1, c1)).astype(np.float32) if c1 else None
    K = k * k * c0 + c1
    w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    res = rng.standard_normal((n, ho, wo, N)).astype(np.float32) if with_res else None
    out = np.empty((n, ho, wo, N), np.float32)
    ms = ctypes.c_float(0)
    ok = lib.boxmot_b200_resnet_conv(x0.ctypes.data, n, h0, w0, c0, k, s, x1.ctypes.data if c1 else None, h1, w1, c1, s1,
                                     w.ctypes.data, N, b.ctypes.data, res.ctypes.data if with_res else None, 1,
                                     out.ctypes.data, ctypes.byref(ms))
    assert ok, _lib.last_error(lib)

    def conv64(x, wk, kk, ss, absval=False):
        xt = torch.from_numpy(x).double().permute(0, 3, 1, 2)
        wt = torch.from_numpy(wk).double().reshape(kk, kk, -1, wk.shape[1]).permute(3, 2, 0, 1)
        if absval:
            xt, wt = xt.abs(), wt.abs()
        return F.conv2d(xt, wt, stride=ss, padding=kk // 2).permute(0, 2, 3, 1).numpy()

    want = conv64(x0, w[: k * k * c0], k, s) + b
    mag = conv64(x0, w[: k * k * c0], k, s, True)
    if c1:
        want = want + conv64(x1, w[k * k * c0:], 1, s1)
        mag = mag + conv64(x1, w[k * k * c0:], 1, s1, True)
    if with_res:
        want = want + res
    want = np.maximum(want, 0)
    err = np.abs(out - want)
    assert (err <= 1e-5 * (mag + 1.0)).all(), f"max err {err.max():.3e}, worst relative {(err / (mag + 1.0)).max():.3e}"
    print(f"conv {case}: max |err| {err.max():.3e}, {ms.value * 1e3:.1f} us")


def test_resnet_every_stage_matches_oracle(tmp_path):
    sd = _state(11)
    reid = _model(tmp_path, sd)
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    x = get_crops(boxes, img, "resize")
    _, want = orn.resnet_forward({k: v.cuda().double() for k, v in sd.items()}, x.cuda().double(), return_stages=True)
    names = ["stem", "pool"] + [f"layer{li + 1}.{j}" for li, nb in enumerate((3, 4, 6, 3)) for j in range(nb)]
    crops = reid.debug_stage(boxes, img, 0).reshape(-1, 256, 128, 3)
    assert np.array_equal(crops, x.permute(0, 2, 3, 1).numpy()), "crop staging must be bit-exact"
    for idx, name in enumerate(names, start=1):
        w = want[name].permute(0, 2, 3, 1).contiguous().cpu().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        err = np.abs(g - w).max()
        assert err < 2e-5 * max(1.0, float(np.abs(w).max())), f"stage {idx} {name}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", ["resnet50", "resnet101", "fc512"])
def test_resnet_matches_reference_golden(tmp_path, case, mode):
    from boxmot_b200.synthetic import make_resnet_state

    z = np.load(GOLDEN / "reid_resnet_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    sd = make_resnet_state(int(z[f"{case}_depth"]), seed=int(z[f"{case}_seed"]), with_fc512=bool(z[f"{case}_fc512"]),
                           num_classes=int(z["num_classes"]))
    reid = _model(tmp_path, sd, case, preprocess=mode)
    assert reid.input_shape == (256, 128) and reid.feature_dim == 2048
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"{case}_features_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("n", [1, 7, 131, 256, 300])
def test_resnet_batch_embeddings_match_oracle(tmp_path, n):
    sd = _state(2)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd).get_features(boxes, img))
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    # a crop's row does not depend on its chunk or on its position in it (300 crops cross the 256-crop chunk)
    tail = slice(max(0, n - 5), n)
    assert np.array_equal(reid.get_features(boxes[tail], img), got[tail])


def test_resnet101_and_resize_pad_match_oracle(tmp_path):
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.concatenate([_boxes(rng, 40, 480, 640), [[5, 5, 300, 470], [-30, -30, -5, -5], [600, 400, 800, 700]]])
    boxes = boxes.astype(np.float32)
    sd = _state(13, depth=101)
    pad = _model(tmp_path, sd, "pad", preprocess="resize_pad")
    _emb_ok(pad.get_features(boxes, img), _DeviceOracle(sd, "resize_pad").get_features(boxes, img))
    _emb_ok(_model(tmp_path, sd, "plain").get_features(boxes, img), _DeviceOracle(sd).get_features(boxes, img))


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_resnet_trackers_match_oracle(tmp_path, kind):
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


def test_resnet_pipelined_device_path_equals_synchronous(tmp_path):
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
        trk = bb.MultiStreamTracker("botsort", n_streams=1, cap_tracks=256, cap_dets=48, feat_dim=2048,
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


def test_create_tracker_with_resnet50_fc512_checkpoint(tmp_path):
    """A seeded checkpoint saved like the released resnet50_fc512_market1501.pt (`state_dict` with `module.` prefixes,
    fc head included) through create_tracker(reid_weights=...): converted once, 2048-d embeddings, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_resnet_state

    sd = make_resnet_state(50, seed=4, with_fc512=True)
    pt = tmp_path / "resnet50_fc512_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    n = sum(len(trk.update(d, img)) for d in frames)
    assert n > 0


def test_reference_abi_botsort_with_resnet_model(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state(6), tmp_path / "abi.b200reid")
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
    dim = ctypes.c_int(0)
    assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 2048
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
