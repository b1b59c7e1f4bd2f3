"""CLIP-ReID ViT-B/16 on the GPU: every new instance of the tensor-core GEMM (the five linear layers, QuickGELU
included, with token rows straddling crops) on its own against float64, the LayerNorm and attention kernels at 129 and
257 tokens, every debug tap against the oracle (oracle.clip.clip_forward), crops bit-exact to the reference's, 1280-d
embeddings against a float64 oracle and the reference golden at 256x128 and 256x256 across the chunk boundary, the
three appearance trackers with on-device CLIP against the oracle trackers, create_tracker with a clip_market1501.pt
checkpoint and the reference ABI.
Embedding bound as for every other backbone: max |delta| <= 1e-4 * ||e||_inf per row, cosine > 0.999999."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import clip as oc
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match


class _DeviceOracle:
    """The oracle's CLIP evaluated by PyTorch on the GPU in float64 on crops staged by the oracle's CPU restatement.
    Test infrastructure only."""

    def __init__(self, sd, preprocess="resize"):
        self.sd = {k: v.cuda() for k, v in oc.double_state(sd).items()}
        self.hw = oc.input_hw(sd)
        self.preprocess = preprocess

    def forward(self, x):
        return torch.cat([oc.clip_forward(self.sd, x[i:i + 32].cuda().double()) for i in range(0, len(x), 32)])

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        f = self.forward(oc.get_crops(xyxys, img, self.preprocess, self.hw)).cpu().numpy()
        return (f / np.linalg.norm(f, axis=-1, keepdims=True)).astype(np.float32)


def _state(seed, vehicle=False):
    from boxmot_b200.synthetic import make_clip_state

    return make_clip_state(seed, vehicle=vehicle)


def _model(tmp_path, sd, name="clip", **kw):
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


# (crops, token rows per crop, K, N, act, residual): the patch embedding (128 / 256 patch rows), in_proj, out_proj +
# residual, c_fc + QuickGELU and c_proj + residual; 129- and 257-row crops make 128-row tiles straddle crops
LINEAR_CASES = [
    (3, 128, 768, 768, 0, False),      # patch embedding, 256x128
    (2, 256, 768, 768, 0, False),      # patch embedding, 256x256
    (3, 129, 768, 2304, 0, False),     # in_proj
    (5, 129, 768, 768, 0, True),       # out_proj + residual
    (3, 129, 768, 3072, 2, False),     # c_fc + QuickGELU
    (1, 257, 768, 3072, 2, False),     # c_fc + QuickGELU, one 257-row crop
    (3, 129, 3072, 768, 0, True),      # c_proj + residual
    (2, 257, 3072, 768, 0, True),      # c_proj + residual, 257 rows
]


@pytest.mark.parametrize("case", LINEAR_CASES, ids=lambda c: f"n{c[0]}_T{c[1]}_K{c[2]}_N{c[3]}_act{c[4]}"
                                                            + ("_res" if c[5] else ""))
def test_clip_linear_kernel_matches_float64(case):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    n, T, K, N, act, with_res = case
    rng = np.random.default_rng(hash(case) & 0xffff)
    x = rng.standard_normal((n, T, 1, K)).astype(np.float32)
    w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    res = rng.standard_normal((n, T, 1, N)).astype(np.float32) if with_res else None
    out = np.empty((n, T, 1, N), np.float32)
    ms = ctypes.c_float(0)
    ok = lib.boxmot_b200_resnet_conv(x.ctypes.data, n, T, 1, K, 1, 1, None, 0, 0, 0, 1, w.ctypes.data, N,
                                     b.ctypes.data, res.ctypes.data if with_res else None, act, out.ctypes.data,
                                     ctypes.byref(ms))
    assert ok, _lib.last_error(lib)
    x64, w64 = x.astype(np.float64).reshape(-1, K), w.astype(np.float64)
    want = x64 @ w64 + b
    mag = np.abs(x64) @ np.abs(w64) + np.abs(b)
    if with_res:
        want = want + res.reshape(-1, N)
    if act == 2:
        want = want / (1.0 + np.exp(-1.702 * want))
    err = np.abs(out.reshape(-1, N) - want)
    assert (err <= 1e-5 * (mag + 1.0)).all(), f"max err {err.max():.3e}"
    print(f"linear {case}: max |err| {err.max():.3e}, {ms.value * 1e3:.1f} us")


@pytest.mark.parametrize("rows", [129, 3 * 257])
def test_clip_layernorm_kernel_matches_float64(rows):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(rows)
    x = (rng.standard_normal((rows, 768)) * 3 + rng.standard_normal((rows, 1)) * 5).astype(np.float32)
    g = rng.uniform(0.5, 1.5, 768).astype(np.float32)
    b = rng.standard_normal(768).astype(np.float32)
    out = np.empty_like(x)
    assert lib.boxmot_b200_vit_layernorm(x.ctypes.data, rows, g.ctypes.data, b.ctypes.data, out.ctypes.data), \
        _lib.last_error(lib)
    want = F.layer_norm(torch.from_numpy(x).double(), (768,), torch.from_numpy(g).double(),
                        torch.from_numpy(b).double(), eps=1e-5).numpy()
    assert np.abs(out - want).max() < 1e-5 * np.abs(want).max()


@pytest.mark.parametrize("n, tokens", [(3, 129), (2, 257), (1, 1), (2, 40)])
def test_clip_attention_kernel_matches_float64(n, tokens):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(tokens)
    qkv = rng.standard_normal((n, tokens, 3 * 768)).astype(np.float32)
    qkv[..., :768] *= 0.4   # scores with a spread of a few units: non-uniform rows
    out = np.empty((n, tokens, 768), np.float32)
    assert lib.boxmot_b200_vit_attention(qkv.ctypes.data, n, tokens, out.ctypes.data), _lib.last_error(lib)
    q, k, v = (torch.from_numpy(z).double().reshape(n, tokens, 12, 64).transpose(1, 2)
               for z in np.split(qkv, 3, axis=-1))
    p = torch.softmax(q @ k.transpose(-1, -2), -1)
    if tokens > 1:
        assert float(p.amax(-1).mean()) > 5.0 / tokens
    want = (p @ v).transpose(1, 2).reshape(n, tokens, 768).numpy()
    assert np.abs(out - want).max() < 2e-5 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("vehicle", [False, True])
def test_clip_every_stage_matches_oracle(tmp_path, vehicle):
    sd = _state(11, vehicle)
    reid = _model(tmp_path, sd)
    hw = (256, 256) if vehicle else (256, 128)
    assert reid.input_shape == hw and reid.feature_dim == 1280
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    x = oc.get_crops(boxes, img, "resize", hw)
    _, want = oc.clip_forward({k: v.cuda() for k, v in oc.double_state(sd).items()}, x.cuda().double(),
                              return_stages=True)
    crops = reid.debug_stage(boxes, img, 0).reshape(-1, *hw, 3)
    assert np.array_equal(crops, x.permute(0, 2, 3, 1).numpy()), "crop staging must be bit-exact"
    # the taps pin the wiring (a wrong operand, offset or order gives O(1) errors); the float32 rounding of the
    # stream grows through the softmax and the LayerNorms (measured: up to 4.5e-5 of the largest entry at the last
    # block), so the bound here is 5e-4 of the largest entry; the 1e-4 precision bound applies to the embeddings
    names = ["patch", "ln_pre"] + [f"block{i}" for i in range(12)] + ["feature"]
    for idx, name in enumerate(names, start=1):
        w = want[name].contiguous().cpu().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        err = np.abs(g - w).max()
        print(f"tap {idx} {name}: max err {err:.3e} of {np.abs(w).max():.3e}")
        assert err < 5e-4 * max(1.0, float(np.abs(w).max())), f"stage {idx} {name}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", ["market", "veri"])
def test_clip_matches_reference_golden(tmp_path, case, mode):
    from boxmot_b200.synthetic import make_clip_state

    z = np.load(GOLDEN / "reid_clip_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    vehicle = bool(z[f"{case}_vehicle"])
    sd = make_clip_state(int(z[f"{case}_seed"]), vehicle=vehicle, num_classes=int(z["num_classes"]))
    reid = _model(tmp_path, sd, case, preprocess=mode)
    hw = (256, 256) if vehicle else (256, 128)
    assert reid.input_shape == hw and reid.feature_dim == 1280
    assert np.array_equal(reid.mean_array, [0.5, 0.5, 0.5]) and np.array_equal(reid.std_array, [0.5, 0.5, 0.5])
    crops = reid.debug_stage(z["boxes"], img, 0).reshape(-1, *hw, 3).transpose(0, 3, 1, 2)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"{case}_crops_sha256_{mode}"])
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, z[f"{case}_features_{mode}"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("n, vehicle", [(1, False), (7, False), (256, False), (300, False), (3, True), (260, True)])
def test_clip_batch_embeddings_match_oracle(tmp_path, n, vehicle):
    sd = _state(2, vehicle)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd).get_features(boxes, img))
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    # a crop's row does not depend on its chunk or on its position in it (300 / 260 crops cross the 256-crop chunk)
    tail = slice(max(0, n - 5), n)
    assert np.array_equal(reid.get_features(boxes[tail], img), got[tail])


def test_clip_resize_pad_matches_oracle(tmp_path):
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.concatenate([_boxes(rng, 20, 480, 640), [[5, 5, 300, 470], [-30, -30, -5, -5], [600, 400, 800, 700]]])
    boxes = boxes.astype(np.float32)
    sd = _state(13, vehicle=True)
    pad = _model(tmp_path, sd, "pad", preprocess="resize_pad")
    _emb_ok(pad.get_features(boxes, img), _DeviceOracle(sd, "resize_pad").get_features(boxes, img))


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_clip_trackers_match_oracle(tmp_path, kind):
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


def test_create_tracker_with_clip_market1501_checkpoint(tmp_path):
    """A seeded checkpoint saved like a CLIP-ReID training checkpoint (`state_dict` with `module.` prefixes, classifier,
    prompt and text keys) through create_tracker(reid_weights=...): converted once, 1280-d embeddings, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_clip_state

    sd = make_clip_state(4)
    pt = tmp_path / "clip_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    n = sum(len(trk.update(d, img)) for d in frames)
    assert n > 0


def test_reference_abi_botsort_with_clip_model(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state(6), tmp_path / "abi.b200reid")
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
    dim = ctypes.c_int(0)
    assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 1280
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
