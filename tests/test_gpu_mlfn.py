"""MLFN on the GPU: the grouped 3x3 kernel, the relu(residual + relu(.)) epilogue of the tensor-core convolution and the
factor-selection module on their own against float64, every stage tap against the oracle (oracle.mlfn.mlfn_forward),
1024-d embeddings against a float64 oracle and the reference-class golden (a strict load and an mlfn_market1501.pt
checkpoint) at chunk boundaries and in both preprocess modes, the three appearance trackers with on-device MLFN against
the oracle trackers, the pipelined device path, create_tracker with an mlfn_market1501.pt checkpoint and the reference
ABI.  Embedding bound as for every other backbone: max |delta| <= 1e-4 * ||e||_inf per row, cosine > 0.999999."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import mlfn as oml
from oracle.reid import get_crops
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match


class _DeviceOracle:
    """The oracle's MLFN evaluated by PyTorch on the GPU in float64 on crops staged by the oracle's CPU restatement.
    Test infrastructure only."""

    def __init__(self, sd, preprocess="resize"):
        self.sd = {k: v.cuda().double() for k, v in sd.items()}
        self.preprocess = preprocess

    def forward(self, x):
        return torch.cat([oml.mlfn_forward(self.sd, x[i:i + 64].cuda().double()) for i in range(0, len(x), 64)])

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        f = self.forward(get_crops(xyxys, img, self.preprocess)).cpu().numpy()
        return (f / np.linalg.norm(f, axis=-1, keepdims=True)).astype(np.float32)


def _state(seed):
    from boxmot_b200.synthetic import make_mlfn_state

    return make_mlfn_state(seed=seed)


def _model(tmp_path, sd, name="mlfn", **kw):
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


# (crops, h, w, group width, stride): every grouped 3x3 of the network (stage s at its input map, the first block of
# stages 2-4 at stride 2), with odd crop counts and a single crop
GROUP_CASES = [(3, 64, 32, 4, 1), (1, 64, 32, 8, 2), (5, 32, 16, 8, 1), (3, 32, 16, 16, 2), (7, 16, 8, 16, 1),
               (1, 16, 8, 32, 2), (9, 8, 4, 32, 1)]


@pytest.mark.parametrize("case", GROUP_CASES, ids=lambda c: f"n{c[0]}_{c[1]}x{c[2]}_gw{c[3]}_s{c[4]}")
def test_mlfn_group_conv_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h, w, gw, s = case
    c = 32 * gw
    rng = np.random.default_rng(hash(case) & 0xffff)
    x = rng.standard_normal((n, h, w, c)).astype(np.float32)
    wt = (rng.standard_normal((9, gw, c)) / np.sqrt(9 * gw)).astype(np.float32)
    b = rng.standard_normal(c).astype(np.float32)
    gates = rng.uniform(0, 1, (n, 32)).astype(np.float32)
    ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
    out = np.empty((n, ho, wo, c), np.float32)
    ok = lib.boxmot_b200_mlfn_group_conv(x.ctypes.data, n, h, w, c, gw, s, wt.ctypes.data, b.ctypes.data,
                                         gates.ctypes.data, out.ctypes.data)
    assert ok, _lib.last_error(lib)
    xt = torch.from_numpy(x).double().permute(0, 3, 1, 2)
    wk = torch.from_numpy(wt).double().reshape(3, 3, gw, c).permute(3, 2, 0, 1)   # [c][gw][3][3]
    conv = F.conv2d(xt, wk, stride=s, padding=1, groups=32)
    mag = F.conv2d(xt.abs(), wk.abs(), stride=s, padding=1, groups=32).permute(0, 2, 3, 1).numpy()
    g = torch.from_numpy(gates).double().repeat_interleave(gw, dim=1)[:, :, None, None]
    want = (F.relu(conv + torch.from_numpy(b).double().view(1, -1, 1, 1)) * g).permute(0, 2, 3, 1).numpy()
    err = np.abs(out - want)
    assert (err <= 1e-5 * (mag + 1.0)).all(), f"max err {err.max():.3e}"


# (crops, h0, w0, c0, N): fm_conv3 of every stage with its residual, straddling crops at 16x8 / 8x4, and fc_s
EPILOGUE_CASES = [(3, 64, 32, 128, 256), (5, 32, 16, 256, 512), (7, 16, 8, 512, 1024), (9, 8, 4, 1024, 2048),
                  (1, 8, 4, 1024, 2048), (7, 1, 1, 512, 1024)]


@pytest.mark.parametrize("case", EPILOGUE_CASES, ids=lambda c: f"n{c[0]}_{c[1]}x{c[2]}x{c[3]}_N{c[4]}")
def test_mlfn_relu_residual_epilogue_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h0, w0, c0, N = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    x = rng.standard_normal((n, h0, w0, c0)).astype(np.float32)
    w = (rng.standard_normal((c0, N)) / np.sqrt(c0)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    res = rng.standard_normal((n, h0, w0, N)).astype(np.float32)
    out = np.empty((n, h0, w0, N), np.float32)
    ok = lib.boxmot_b200_resnet_conv(x.ctypes.data, n, h0, w0, c0, 1, 1, None, 0, 0, 0, 1, w.ctypes.data, N,
                                     b.ctypes.data, res.ctypes.data, 3, out.ctypes.data, None)
    assert ok, _lib.last_error(lib)
    x64, w64 = x.astype(np.float64), w.astype(np.float64)
    want = np.maximum(res + np.maximum(x64 @ w64 + b, 0), 0)
    mag = np.abs(x64) @ np.abs(w64)
    err = np.abs(out - want)
    assert (err <= 1e-5 * (mag + 1.0)).all(), f"max err {err.max():.3e}"


# (crops, h, w, c, f0, f1): the FSM of every stage (block 0's 64-channel input included), odd counts and one crop
FSM_CASES = [(3, 64, 32, 64, 128, 64), (1, 64, 32, 256, 128, 64), (5, 32, 16, 512, 256, 128),
             (7, 16, 8, 1024, 512, 128), (9, 8, 4, 2048, 512, 128), (1, 8, 4, 2048, 512, 128)]


@pytest.mark.parametrize("case", FSM_CASES, ids=lambda c: f"n{c[0]}_{c[1]}x{c[2]}x{c[3]}_f{c[4]}_{c[5]}")
def test_mlfn_fsm_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h, w, c, f0, f1 = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    x = np.abs(rng.standard_normal((n, h, w, c))).astype(np.float32)
    w1 = (rng.standard_normal((c, f0)) / np.sqrt(c)).astype(np.float32)
    w2 = (rng.standard_normal((f0, f1)) / np.sqrt(f0)).astype(np.float32)
    w3 = (rng.standard_normal((f1, 32)) / np.sqrt(f1)).astype(np.float32)
    b1, b2, b3 = (0.1 * rng.standard_normal(k).astype(np.float32) for k in (f0, f1, 32))
    out = np.empty((n, 32), np.float32)
    ok = lib.boxmot_b200_mlfn_fsm(x.ctypes.data, n, h, w, c, w1.ctypes.data, b1.ctypes.data, f0, w2.ctypes.data,
                                  b2.ctypes.data, f1, w3.ctypes.data, b3.ctypes.data, out.ctypes.data)
    assert ok, _lib.last_error(lib)
    p = x.astype(np.float64).mean(axis=(1, 2))
    h1 = np.maximum(p @ w1 + b1, 0)
    h2 = np.maximum(h1 @ w2 + b2, 0)
    z = h2 @ w3 + b3
    want = 1 / (1 + np.exp(-z))
    mag = np.abs(h2) @ np.abs(w3) + 1.0
    err = np.abs(out - want)
    assert (err <= 1e-5 * mag).all(), f"max err {err.max():.3e}"
    # a crop's gates do not depend on the other crops of the call
    one = np.empty((1, 32), np.float32)
    xl = np.ascontiguousarray(x[-1:])
    assert lib.boxmot_b200_mlfn_fsm(xl.ctypes.data, 1, h, w, c, w1.ctypes.data, b1.ctypes.data, f0, w2.ctypes.data,
                                    b2.ctypes.data, f1, w3.ctypes.data, b3.ctypes.data, one.ctypes.data)
    assert np.array_equal(one[0], out[-1])


def test_mlfn_every_stage_matches_oracle(tmp_path):
    sd = _state(11)
    reid = _model(tmp_path, sd)
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    x = get_crops(boxes, img, "resize")
    _, want = oml.mlfn_forward({k: v.cuda().double() for k, v in sd.items()}, x.cuda().double(), return_stages=True)
    names = ["stem", "pool"] + [f"feature.{i}" for i in range(16)] + ["s_hat", "v"]
    crops = reid.debug_stage(boxes, img, 0).reshape(-1, 256, 128, 3)
    assert np.array_equal(crops, x.permute(0, 2, 3, 1).numpy()), "crop staging must be bit-exact"
    for idx, name in enumerate(names, start=1):
        t = want[name]
        w = (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).contiguous().cpu().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        err = np.abs(g - w).max()
        # v is the un-normalised embedding: fc_x contracts 2048 pooled channels, so it carries the maps' float32 error
        # amplified (2.3e-5 of its largest entry measured); it gets the embedding bound, every map and s_hat 2e-5
        tol = 1e-4 if name == "v" else 2e-5
        assert err < tol * max(1.0, float(np.abs(w).max())), f"stage {idx} {name}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", ["strict", "checkpoint"])
def test_mlfn_matches_reference_golden(tmp_path, case, mode):
    from boxmot_b200.synthetic import make_mlfn_state

    z = np.load(GOLDEN / "reid_mlfn_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    sd = make_mlfn_state(seed=int(z[f"{case}_seed"]), num_classes=int(z["num_classes"]))
    reid = _model(tmp_path, sd, case, preprocess=mode)
    assert reid.input_shape == (256, 128) and reid.feature_dim == 1024
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"{case}_features_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("n", [1, 7, 131, 256, 300])
def test_mlfn_batch_embeddings_match_oracle(tmp_path, n):
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


def test_mlfn_resize_pad_matches_oracle(tmp_path):
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.concatenate([_boxes(rng, 40, 480, 640), [[5, 5, 300, 470], [-30, -30, -5, -5], [600, 400, 800, 700]]])
    boxes = boxes.astype(np.float32)
    sd = _state(13)
    pad = _model(tmp_path, sd, "pad", preprocess="resize_pad")
    _emb_ok(pad.get_features(boxes, img), _DeviceOracle(sd, "resize_pad").get_features(boxes, img))


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_mlfn_trackers_match_oracle(tmp_path, kind):
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


def test_mlfn_pipelined_device_path_equals_synchronous(tmp_path):
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
        trk = bb.MultiStreamTracker("botsort", n_streams=1, cap_tracks=256, cap_dets=48, feat_dim=1024,
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


def test_create_tracker_with_mlfn_checkpoint(tmp_path):
    """A seeded checkpoint saved like the released mlfn_market1501.pt (`state_dict` with `module.` prefixes, classifier
    included) through create_tracker(reid_weights=...): converted once, 1024-d embeddings, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_mlfn_state

    sd = make_mlfn_state(seed=4)
    pt = tmp_path / "mlfn_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    n = sum(len(trk.update(d, img)) for d in frames)
    assert n > 0


def test_reference_abi_botsort_with_mlfn_model(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state(6), tmp_path / "abi.b200reid")
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
    dim = ctypes.c_int(0)
    assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 1024
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
