"""HACNN on the GPU: each new kernel on its own against float64 (the tensor-core ConvBlock's slice store, the stem, both
pools at even and odd sizes, the attention with theta, the STN resample at the three levels with regions partly off
the map, the head), every stage tap against the oracle (oracle.hacnn.hacnn_forward), 1024-d embeddings against a
float64 oracle and the reference-class golden (a strict load and a hacnn_market1501.pt checkpoint) at chunk boundaries
and in both preprocess modes, the three appearance trackers with on-device HACNN against the oracle trackers, the
pipelined device path, create_tracker with a hacnn_market1501.pt checkpoint and the reference ABI.  Embedding bound as
for every other backbone: max |delta| <= 1e-4 * ||e||_inf per row, cosine > 0.999999."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import hacnn as oha
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match


class _DeviceOracle:
    """The oracle's HACNN evaluated by PyTorch on the GPU in float64 on crops staged by the oracle's CPU restatement.
    Test infrastructure only."""

    def __init__(self, sd, preprocess="resize"):
        self.sd = {k: v.cuda().double() for k, v in sd.items()}
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        x = oha.get_crops(xyxys, img, self.preprocess)
        v = torch.cat([oha.hacnn_forward(self.sd, x[i:i + 64].cuda().double()) for i in range(0, len(x), 64)])
        return oha.embed(v).cpu().numpy().astype(np.float32)


def _state(seed):
    from boxmot_b200.synthetic import make_hacnn_state

    return make_hacnn_state(seed=seed)


def _model(tmp_path, sd, name="hacnn", **kw):
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


def _nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a)).double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().numpy()


# (crops, h, w, c0, k, stride, N, out_ld, out_off): the stream shapes of the network (mid widths 32 / 64 / 96, the
# 2 x mid max-pool streams, odd local maps 24x28 -> 12x14 -> 6x7 -> 3x4) and the heads over a [crops] x 1 map
CONV_CASES = [(3, 80, 32, 32, 1, 1, 32, 128, 0), (2, 80, 32, 32, 3, 1, 32, 128, 96), (5, 80, 32, 128, 3, 2, 32, 128, 32),
              (3, 40, 16, 128, 1, 1, 64, 128, 64), (4, 40, 16, 64, 3, 2, 64, 256, 64), (3, 20, 8, 256, 1, 1, 96, 384, 288),
              (2, 20, 8, 96, 3, 2, 96, 384, 96), (9, 12, 14, 128, 1, 1, 128, 256, 128), (7, 6, 7, 96, 3, 2, 96, 384, 0),
              (5, 3, 4, 256, 1, 1, 192, 384, 192), (6, 24, 28, 32, 3, 2, 32, 128, 32), (7, 1, 1, 1536, 1, 1, 512, 1024, 512)]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n{}_{}x{}x{}_k{}s{}_N{}_ld{}+{}".format(*c))
def test_hacnn_conv_slice_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h, w, c0, k, s, N, ld, o = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    x = rng.standard_normal((n, h, w, c0)).astype(np.float32)
    x[rng.uniform(size=x.shape) < 0.2] = 0
    wt = (rng.standard_normal((k * k * c0, N)) / np.sqrt(k * k * c0)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
    for off, count in ((0, n), (1, n - 1)):   # the window skips crop 0 in the second call (a chunk starting at 1)
        out = np.full((n, ho, wo, ld), np.nan, np.float32)
        ok = lib.boxmot_b200_hacnn_conv(x.ctypes.data, n, off, count, h, w, c0, k, s, wt.ctypes.data, N, b.ctypes.data,
                                        out.ctypes.data, ld, o)
        assert ok, _lib.last_error(lib)
        live = count - off
        wk = torch.from_numpy(wt).double().reshape(k, k, c0, N).permute(3, 2, 0, 1)
        xt = _nchw(x[:live])
        want = _nhwc(F.relu(F.conv2d(xt, wk, torch.from_numpy(b).double(), stride=s, padding=k // 2)))
        mag = _nhwc(F.conv2d(xt.abs(), wk.abs(), stride=s, padding=k // 2)) + np.abs(b)
        err = np.abs(out[:live, ..., o:o + N] - want)
        assert (err <= 1e-5 * (mag + 1.0)).all(), f"max err {np.nanmax(err):.3e}"
        rest = np.delete(out, np.s_[o:o + N], axis=3)   # the other channels and the crops outside the window
        assert np.isnan(rest).all() and np.isnan(out[live:]).all()


def test_hacnn_stem_matches_float64():
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(5)
    n = 3
    x = rng.standard_normal((n, 160, 64, 3)).astype(np.float32)
    wt = rng.standard_normal((27, 32)).astype(np.float32)
    b = rng.standard_normal(32).astype(np.float32)
    out = np.full((n, 80, 32, 32), np.nan, np.float32)
    assert lib.boxmot_b200_hacnn_map(0, x.ctypes.data, n, 0, n - 1, 160, 64, 3, wt.ctypes.data, b.ctypes.data,
                                     out.ctypes.data), _lib.last_error(lib)
    wk = torch.from_numpy(wt).double().reshape(3, 3, 3, 32).permute(3, 2, 0, 1)
    want = _nhwc(F.relu(F.conv2d(_nchw(x), wk, torch.from_numpy(b).double(), stride=2, padding=1)))
    mag = _nhwc(F.conv2d(_nchw(x).abs(), wk.abs(), stride=2, padding=1)) + np.abs(b)
    assert (np.abs(out[:2] - want[:2]) <= 1e-6 * (mag[:2] + 1)).all()
    assert np.isnan(out[2]).all()


# (crops, h, w, c, op): the average pools (stride 1) and max pools (stride 2) of the network, odd local maps included
POOL_CASES = [(3, 80, 32, 32, 1), (2, 40, 16, 128, 1), (3, 20, 8, 256, 1), (3, 80, 32, 128, 2), (2, 40, 16, 256, 2),
              (3, 20, 8, 384, 2), (9, 24, 28, 32, 2), (7, 12, 14, 128, 2), (5, 6, 7, 256, 2)]


@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "n{}_{}x{}x{}_op{}".format(*c))
def test_hacnn_pools_match_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h, w, c, op = case
    x = np.random.default_rng(hash(case) & 0xffff).standard_normal((n, h, w, c)).astype(np.float32)
    ho, wo = ((h - 1) // 2 + 1, (w - 1) // 2 + 1) if op == 2 else (h, w)
    out = np.full((n, ho, wo, c), np.nan, np.float32)
    assert lib.boxmot_b200_hacnn_map(op, x.ctypes.data, n, 0, n, h, w, c, None, None, out.ctypes.data), \
        _lib.last_error(lib)
    xt = _nchw(x)
    if op == 2:
        assert np.array_equal(out, _nhwc(F.max_pool2d(xt, 3, 2, 1)).astype(np.float32))
    else:
        want = _nhwc(F.avg_pool2d(xt, 3, 1, 1))
        assert np.abs(out - want).max() <= 1e-6 * (1 + np.abs(x).max())


def _attn_params(rng, c):
    r = c // 16
    parts = [np.concatenate([rng.standard_normal(9) / 3, [0.1], [1.5, 0.2]]), rng.standard_normal((c, r)) / np.sqrt(c),
             0.1 * rng.standard_normal(r), rng.standard_normal((r, c)) / np.sqrt(r), 0.1 * rng.standard_normal(c),
             rng.standard_normal((c, c)) / np.sqrt(c), rng.standard_normal(c) * 0.5, 2 * rng.standard_normal((c, 8)) / np.sqrt(c),
             0.3 * rng.standard_normal(8)]
    flat = np.concatenate([np.pad(np.ravel(p), (0, (-np.size(p)) % 4)) for p in parts]).astype(np.float32)
    return [np.asarray(p, np.float32) for p in parts], flat


@pytest.mark.parametrize("case", [(3, 40, 16, 128, 0), (2, 20, 8, 256, 1), (5, 10, 4, 384, 2)],
                         ids=lambda c: "n{}_{}x{}x{}_level{}".format(*c))
def test_hacnn_attention_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, h, w, c, level = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    x = np.abs(rng.standard_normal((n, h, w, c))).astype(np.float32)
    (sp, w1, b1, w2, b2, wv, bv, wfc, bfc), flat = _attn_params(rng, c)
    out = np.full_like(x, np.nan)
    s, v = np.full((n, h * w), np.nan, np.float32), np.full((n, c), np.nan, np.float32)
    theta = np.full((n, 24), np.nan, np.float32)
    assert lib.boxmot_b200_hacnn_attention(x.ctypes.data, n, 0, n - 1, h, w, c, level, flat.ctypes.data,
                                           out.ctypes.data, s.ctypes.data, v.ctypes.data, theta.ctypes.data), \
        _lib.last_error(lib)
    d = {k: torch.from_numpy(np.asarray(a, np.float64)) for k, a in
         dict(sp=sp, w1=w1, b1=b1, w2=w2, b2=b2, wv=wv, bv=bv, wfc=wfc, bfc=bfc).items()}
    xt = _nchw(x[:n - 1])
    m = F.conv2d(xt.mean(1, keepdim=True), d["sp"][:9].view(1, 1, 3, 3), d["sp"][9:10], stride=2, padding=1)
    m = F.interpolate(F.relu(m), scale_factor=2, mode="bilinear", align_corners=True)
    s64 = F.relu(d["sp"][10] * m + d["sp"][11])
    g = xt.mean(dim=(2, 3))
    ch = F.relu(F.relu(g @ d["w1"] + d["b1"]) @ d["w2"] + d["b2"])
    v64 = ch @ d["wv"]
    att = torch.sigmoid(F.relu(s64 * v64[:, :, None, None] + d["bv"][None, :, None, None]))
    th = torch.tanh(g @ d["wfc"] + d["bfc"]).numpy()
    assert np.abs(s[:n - 1] - s64.flatten(1).numpy()).max() < 1e-5 * (1 + s64.abs().max().item())
    assert np.abs(v[:n - 1] - v64.numpy()).max() < 1e-5 * (1 + (ch.abs() @ d["wv"].abs()).max().item())
    assert np.abs(theta[:n - 1, 8 * level:8 * level + 8] - th).max() < 1e-5
    assert np.abs(out[:n - 1] - _nhwc(xt * att)).max() < 2e-6 * (1 + np.abs(x).max())
    keep = np.delete(theta, np.s_[8 * level:8 * level + 8], axis=1)
    assert np.isnan(keep).all() and np.isnan(theta[n - 1]).all() and np.isnan(s[n - 1]).all()
    assert np.array_equal(out[n - 1], x[n - 1])   # the window leaves the last crop's map as it was


# (crops, source h, w, c, level, local h, w): the three STN levels
STN_CASES = [(3, 80, 32, 32, 0, 24, 28), (2, 40, 16, 128, 1, 12, 14), (5, 20, 8, 256, 2, 6, 7)]


@pytest.mark.parametrize("case", STN_CASES, ids=lambda c: "n{}_{}x{}x{}_level{}".format(*c))
def test_hacnn_stn_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, H, W, C, level, lh, lw = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    src = rng.standard_normal((n, H, W, C)).astype(np.float32)
    theta = np.full((n, 24), np.nan, np.float32)
    # regions off centre, partly off the map at every side, one centred
    th = np.array([[0.7, -0.9], [-0.6, -0.2], [0.0, 0.3], [0.35, 0.95]], np.float32) + \
        0.05 * rng.standard_normal((n, 4, 2)).astype(np.float32)
    theta[:, 8 * level:8 * level + 8] = th.reshape(n, 8)
    prev = rng.standard_normal((n, 4, lh, lw, C)).astype(np.float32) if level else None
    out = np.full((n, 4, lh, lw, C), np.nan, np.float32)
    assert lib.boxmot_b200_hacnn_stn(src.ctypes.data, n, 0, n, H, W, C, theta.ctypes.data, level,
                                     None if prev is None else prev.ctypes.data, lh, lw, out.ctypes.data), \
        _lib.last_error(lib)
    st = _nchw(src)
    for r in range(4):
        t = F.interpolate(oha.stn(st, torch.from_numpy(th[:, r]).double()), (lh, lw), mode="bilinear",
                          align_corners=True)
        want = _nhwc(t) + (prev[:, r] if prev is not None else 0)
        assert np.abs(out[:, r] - want).max() < 1e-5 * (1 + np.abs(src).max()), f"region {r}"
    # some samples fall outside the map: the regions really leave it
    assert (np.abs(th[..., 0]) > 0.5).any() and (np.abs(th[..., 1]) > 0.75).any()


def test_hacnn_head_matches_float64():
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(9)
    n = 5
    x3 = np.abs(rng.standard_normal((n, 40, 384))).astype(np.float32)
    loc = np.abs(rng.standard_normal((n, 4, 12, 384))).astype(np.float32)
    wg = (rng.standard_normal((384, 512)) / np.sqrt(384)).astype(np.float32)
    wl = (rng.standard_normal((1536, 512)) / np.sqrt(1536)).astype(np.float32)
    bg, bl = (0.1 * rng.standard_normal(512).astype(np.float32) for _ in range(2))
    rows = np.array([4, 0, 3, 1, 2], np.int32)
    out = np.full((6, 1024), np.nan, np.float32)
    v = np.full((n, 1024), np.nan, np.float32)
    assert lib.boxmot_b200_hacnn_head(x3.ctypes.data, n, 0, n, 40, loc.ctypes.data, 12, wg.ctypes.data,
                                      bg.ctypes.data, wl.ctypes.data, bl.ctypes.data, rows.ctypes.data, 6,
                                      out.ctypes.data, v.ctypes.data), _lib.last_error(lib)
    pg = x3.astype(np.float64).mean(1)
    pl = loc.astype(np.float64).mean(2).reshape(n, -1)
    v64 = np.concatenate([np.maximum(pg @ wg + bg, 0), np.maximum(pl @ wl + bl, 0)], 1)
    assert np.abs(v - v64).max() < 1e-5 * (1 + np.abs(v64).max())
    e = oha.embed(torch.from_numpy(v64)).numpy()
    assert np.abs(out[rows] - e).max() < 1e-6
    assert np.isnan(out[5]).all()


def test_hacnn_every_stage_matches_oracle(tmp_path):
    sd = _state(11)
    reid = _model(tmp_path, sd)
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    x = oha.get_crops(boxes, img, "resize")
    _, want = oha.hacnn_forward({k: v.cuda().double() for k, v in sd.items()}, x.cuda().double(), return_stages=True)
    crops = reid.debug_stage(boxes, img, 0).reshape(-1, 160, 64, 3)
    assert np.array_equal(crops, x.permute(0, 2, 3, 1).numpy()), "crop staging must be bit-exact"
    names = ["stem", "x1_out", "x2_out", "x3_out", "local1", "local2", "local3", "theta", "v"]
    for idx, name in enumerate(names, start=1):
        t = want[name]
        if t.dim() == 5:   # (N, 4, C, h, w) -> [region][h][w][C]
            t = t.permute(0, 1, 3, 4, 2)
        elif t.dim() == 4:
            t = t.permute(0, 2, 3, 1)
        w = t.contiguous().cpu().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        err = np.abs(g - w).max() / max(1.0, float(np.abs(w).max()))
        print(f"stage {idx} {name}: max err / max(1, ||w||inf) = {err:.2e}")
        # the global maps, theta and the head row get the embedding bound.  The local maps sample the previous level at
        # x + tx W / 2: theta's float32 error (~1e-5) moves every sample by up to 1e-5 x 16 px across maps whose
        # gradient reaches ~10 per pixel, so they carry ~1e-3 relative error (5.5e-4 measured for local1; PyTorch's
        # own float32 forward is 3.4e-5 off here).  The head row v carries that error through fc_local (1.3e-4
        # measured).  The normalised embeddings stay within 1e-4, checked below
        tol = 3e-3 if name.startswith("local") else (3e-4 if name == "v" else 1e-4)
        assert err < tol, f"stage {idx} {name}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", ["strict", "checkpoint"])
def test_hacnn_matches_reference_golden(tmp_path, case, mode):
    from boxmot_b200.synthetic import make_hacnn_state

    z = np.load(GOLDEN / "reid_hacnn_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    sd = make_hacnn_state(seed=int(z[f"{case}_seed"]), num_classes=int(z["num_classes"]))
    reid = _model(tmp_path, sd, case, preprocess=mode)
    assert reid.input_shape == (160, 64) and reid.feature_dim == 1024
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"{case}_features_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 300])
def test_hacnn_batch_embeddings_match_oracle(tmp_path, n):
    sd = _state(2)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd).get_features(boxes, img))
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    # a crop's row does not depend on its chunk or on its position in it (257 and 300 crops cross the 256-crop chunk)
    tail = slice(max(0, n - 5), n)
    assert np.array_equal(reid.get_features(boxes[tail], img), got[tail])


def test_hacnn_resize_pad_matches_oracle(tmp_path):
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.concatenate([_boxes(rng, 40, 480, 640), [[5, 5, 300, 470], [-30, -30, -5, -5], [600, 400, 800, 700]]])
    boxes = boxes.astype(np.float32)
    sd = _state(13)
    pad = _model(tmp_path, sd, "pad", preprocess="resize_pad")
    _emb_ok(pad.get_features(boxes, img), _DeviceOracle(sd, "resize_pad").get_features(boxes, img))


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_hacnn_trackers_match_oracle(tmp_path, kind):
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


def test_hacnn_pipelined_device_path_equals_synchronous(tmp_path):
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


def test_create_tracker_with_hacnn_checkpoint(tmp_path):
    """A seeded checkpoint saved like the released hacnn_market1501.pt (`state_dict` with `module.` prefixes,
    classifiers included) through create_tracker(reid_weights=...): converted once, 1024-d embeddings, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_hacnn_state

    sd = make_hacnn_state(seed=4)
    pt = tmp_path / "hacnn_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    n = sum(len(trk.update(d, img)) for d in frames)
    assert n > 0


def test_reference_abi_botsort_with_hacnn_model(tmp_path):
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
