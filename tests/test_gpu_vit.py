"""ViT-Nano / ViT-Tiny on the GPU: the new tensor-core GEMM shapes (patch embedding at 128 and 310 patch rows, qkv,
proj + residual, fc1 + exact GELU, fc2 + residual, with token rows straddling 129- and 311-row crops) on their own
against float64, the 192-wide LayerNorm, the AIN norm, the attention at 1 / 40 / 129 / 311 tokens and every head
against float64, every debug tap against the oracle (tests/vit_oracle.py), all six variants against the reference
golden and a float64 oracle across the chunk boundary, the three appearance trackers with on-device ViT against the
oracle trackers, the pipelined path, create_tracker with a trainer-format checkpoint and the reference ABI.
Embedding bound as for every other backbone: max |delta| <= 1e-4 * ||e||_inf per row, cosine > 0.999999."""
import ctypes
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from boxmot_b200.weights import VIT_VARIANTS
from tests import vit_oracle as ov
from tests.common import BOTSORT_YAML, GOLDEN, assert_rows_match

VARIANTS = tuple(VIT_VARIANTS)


class _DeviceOracle:
    """The oracle's ViT evaluated by PyTorch on the GPU in float64 on crops staged by the oracle's CPU restatement."""

    def __init__(self, sd, variant, preprocess="resize"):
        self.sd = {k: v.cuda() for k, v in ov.double_state(sd).items()}
        self.variant = variant
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        x = ov.get_crops(xyxys, img, self.preprocess, ov.input_hw(self.variant))
        f = torch.cat([ov.vit_forward(self.sd, self.variant, x[i:i + 64].cuda().double())
                       for i in range(0, len(x), 64)]).cpu().numpy()
        return (f / np.linalg.norm(f, axis=-1, keepdims=True)).astype(np.float32)


def _state(variant, seed):
    from boxmot_b200.synthetic import make_vit_state

    return make_vit_state(variant, seed)


def _model(tmp_path, sd, name="vit", **kw):
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


# (crops, token rows per crop, K, N, act, residual); 129- and 311-row crops make 128-row tiles straddle crops
LINEAR_CASES = [
    (3, 128, 768, 192, 0, False),      # patch embedding, 256x128
    (2, 310, 768, 192, 0, False),      # patch embedding, 384x128 at stride 12
    (3, 129, 192, 576, 0, False),      # qkv
    (2, 311, 192, 576, 0, False),
    (5, 129, 192, 192, 0, True),       # proj + residual
    (3, 129, 192, 768, 4, False),      # fc1 + GELU
    (2, 311, 192, 768, 4, False),
    (1, 40, 192, 192, 4, False),       # GELU on a 64-wide tile instance
    (3, 129, 768, 192, 0, True),       # fc2 + residual
    (2, 311, 768, 192, 0, True),
]


@pytest.mark.parametrize("case", LINEAR_CASES, ids=lambda c: f"n{c[0]}_T{c[1]}_K{c[2]}_N{c[3]}_act{c[4]}"
                                                            + ("_res" if c[5] else ""))
def test_vit_linear_kernel_matches_float64(case):
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
    if act == 4:
        want = F.gelu(torch.from_numpy(want)).numpy()
    err = np.abs(out.reshape(-1, N) - want)
    assert (err <= 1e-5 * (mag + 1.0)).all(), f"max err {err.max():.3e}"
    print(f"linear {case}: max |err| {err.max():.3e}, {ms.value * 1e3:.1f} us")


@pytest.mark.parametrize("rows", [129, 3 * 311])
def test_vit_layernorm192_kernel_matches_float64(rows):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(rows)
    x = (rng.standard_normal((rows, 192)) * 3 + rng.standard_normal((rows, 1)) * 5).astype(np.float32)
    g = rng.uniform(0.5, 1.5, 192).astype(np.float32)
    b = rng.standard_normal(192).astype(np.float32)
    out = np.empty_like(x)
    assert lib.boxmot_b200_vits_layernorm(x.ctypes.data, rows, g.ctypes.data, b.ctypes.data, out.ctypes.data), \
        _lib.last_error(lib)
    want = F.layer_norm(torch.from_numpy(x).double(), (192,), torch.from_numpy(g).double(),
                        torch.from_numpy(b).double(), eps=1e-5).numpy()
    assert np.abs(out - want).max() < 1e-5 * np.abs(want).max()


@pytest.mark.parametrize("n, tokens", [(3, 129), (1, 1), (2, 40)])
def test_vit_ain_kernel_matches_float64(n, tokens):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(tokens)
    # per-channel offsets and scales that IN removes and LN does not
    x = (rng.standard_normal((n, tokens, 192)) * rng.uniform(0.5, 3, 192) + rng.standard_normal(192) * 4)
    x = x.astype(np.float32)
    a, b, s = (rng.standard_normal(192).astype(np.float32) for _ in range(3))
    out = np.empty_like(x)
    assert lib.boxmot_b200_vits_ain(x.ctypes.data, n, tokens, a.ctypes.data, b.ctypes.data, s.ctypes.data,
                                    out.ctypes.data), _lib.last_error(lib)
    t = torch.from_numpy(x).double()
    mu, var = t.mean(1, keepdim=True), t.var(1, unbiased=False, keepdim=True)
    xin = (t - mu) / torch.sqrt(var + 1e-5)   # InstanceNorm1d over the tokens (also defined for a single token)
    want = (torch.from_numpy(a).double() * xin + torch.from_numpy(b).double() * F.layer_norm(t, (192,), eps=1e-5)
            + torch.from_numpy(s).double()).numpy()
    mag = np.abs(a).max() * (np.abs(xin.numpy()).max() + 1) + np.abs(b).max() * 4
    assert np.abs(out - want).max() < 1e-5 * mag


@pytest.mark.parametrize("n, tokens", [(3, 129), (2, 311), (1, 1), (2, 40)])
def test_vit_attention192_kernel_matches_float64(n, tokens):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    rng = np.random.default_rng(tokens)
    qkv = rng.standard_normal((n, tokens, 3 * 192)).astype(np.float32)
    qkv[..., :192] *= 0.4   # scores with a spread of a few units: non-uniform rows
    out = np.empty((n, tokens, 192), np.float32)
    assert lib.boxmot_b200_vit_attention_width(qkv.ctypes.data, n, tokens, 192, out.ctypes.data), _lib.last_error(lib)
    q, k, v = (torch.from_numpy(z).double().reshape(n, tokens, 3, 64).transpose(1, 2)
               for z in np.split(qkv, 3, axis=-1))
    p = torch.softmax(q @ k.transpose(-1, -2), -1)
    if tokens > 1:
        assert float(p.amax(-1).mean()) > 5.0 / tokens
    want = (p @ v).transpose(1, 2).reshape(n, tokens, 192).numpy()
    assert np.abs(out - want).max() < 2e-5 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("variant", ["vit_nano", "vit_nano_ain_os", "vit_tiny", "vit_tiny_parts", "vit_tiny_parts3"])
def test_vit_head_kernel_matches_float64(tmp_path, variant):
    """The head block of the blob on random final-norm outputs: the kernel's row before and after the L2 norm against
    the float64 walk of the same weights."""
    from boxmot_b200 import _lib
    from boxmot_b200.weights import export_blob, read_blob

    lib = _lib.require_device()
    header, payload = read_blob(export_blob(_state(variant, 8), tmp_path / "h.b200reid"))
    feat, (gh, gw, pool, proj) = header[7], (header[11], header[12], header[14], header[15])
    n_hw = (4 * 2 * 192 + 192 * 12 + 12 + 12 * 192 + 192 + 2 * 192) if pool == 1 else (
        (1 + (pool if pool >= 2 else 0)) * (192 * proj + proj) if proj else 2 * 192)
    hw = np.ascontiguousarray(payload[-n_hw:])
    n = 5
    rng = np.random.default_rng(3)
    x = rng.standard_normal((n, 1 + gh * gw, 192)).astype(np.float32)
    raw, nrm = np.empty((n, feat), np.float32), np.empty((n, feat), np.float32)
    for normalise, out in ((0, raw), (1, nrm)):
        assert lib.boxmot_b200_vits_head(x.ctypes.data, n, gh, gw, pool, proj, hw.ctypes.data, n_hw, normalise,
                                         out.ctypes.data), _lib.last_error(lib)
    want = _head64(torch.from_numpy(x).double(), torch.from_numpy(hw.astype(np.float64)), gh, gw, pool, proj).numpy()
    assert np.abs(raw - want).max() < 1e-5 * max(1.0, np.abs(want).max())
    want_n = want / np.linalg.norm(want, axis=1, keepdims=True)
    assert np.abs(nrm - want_n).max() < 1e-5 * np.abs(want_n).max()


def _head64(h, hw, gh, gw, pool, proj):
    """Float64 restatement of the head block (weights.fold_vit's head layout) on final-norm outputs h (n, T, 192)."""
    o, d, n = 0, 192, h.shape[0]

    def take(*shape):
        nonlocal o
        k = int(np.prod(shape))
        t = hw[o:o + k].reshape(shape)
        o += k
        return t

    ln = lambda t: F.layer_norm(t, (d,), eps=1e-5)   # noqa: E731
    if pool == 1:
        pm = h[:, 1:].mean(1)
        gs = [(take(d), take(d)) for _ in range(4)]
        w1, b1, w2, b2 = take(d, 12), take(12), take(12, d), take(d)
        f = 0
        for g, bb in gs:
            qv = ln(pm) * g + bb
            f = f + torch.sigmoid(torch.relu(qv @ w1 + b1) @ w2 + b2) * qv
        return f * take(d) + take(d)
    if not proj:
        return h[:, 0] * take(d) + take(d)
    vecs = [h[:, 0]]
    sp = h[:, 1:].reshape(n, gh, gw, d)
    for i in range(pool if pool >= 2 else 0):
        r0 = i * (gh // pool)
        r1 = gh if i == pool - 1 else r0 + gh // pool
        vecs.append(sp[:, r0:r1].mean((1, 2)))
    return torch.cat([v @ take(d, proj) + take(proj) for v in vecs], 1)


@pytest.mark.parametrize("variant", ["vit_nano_ain_os", "vit_tiny_parts3"])
def test_vit_every_stage_matches_oracle(tmp_path, variant):
    sd = _state(variant, 11)
    reid = _model(tmp_path, sd)
    hw = ov.input_hw(variant)
    assert reid.input_shape == hw
    img = np.random.default_rng(0).integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    x = ov.get_crops(boxes, img, "resize", hw)
    _, want = ov.vit_forward({k: v.cuda() for k, v in ov.double_state(sd).items()}, variant, x.cuda().double(),
                             return_stages=True)
    crops = reid.debug_stage(boxes, img, 0).reshape(-1, *hw, 3)
    assert np.array_equal(crops, x.permute(0, 2, 3, 1).numpy()), "crop staging must be bit-exact"
    depth = VIT_VARIANTS[variant][0]
    names = ["patch", "tokens"] + [f"block{i}" for i in range(depth)] + ["norm", "feature"]
    for idx, name in enumerate(names, start=1):
        w = want[name].contiguous().cpu().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        err = np.abs(g - w).max()
        print(f"tap {idx} {name}: max err {err:.3e} of {np.abs(w).max():.3e}")
        assert err < 5e-4 * max(1.0, float(np.abs(w).max())), f"stage {idx} {name}: max err {err:.3e}"


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_vit_matches_reference_golden(tmp_path, variant, mode):
    from boxmot_b200.synthetic import make_vit_state

    z = np.load(GOLDEN / "reid_vit_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    sd = make_vit_state(variant, int(z[f"{variant}_seed"]), num_classes=int(z["num_classes"]))
    pt = tmp_path / f"{variant}_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_name": variant}, pt)
    from boxmot_b200.reid import B200ReID

    reid = B200ReID(pt, preprocess=mode)
    hw = ov.input_hw(variant)
    want = z[f"{variant}_features_{mode}"]
    assert reid.input_shape == hw and reid.feature_dim == want.shape[1]
    crops = reid.debug_stage(z["boxes"], img, 0).reshape(-1, *hw, 3).transpose(0, 3, 1, 2)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"{variant}_crops_sha256_{mode}"])
    feats = reid.get_features(z["boxes"], img)
    _emb_ok(feats, want)
    _emb_ok(feats, ov.get_features(sd, variant, z["boxes"], img, mode))
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5


@pytest.mark.parametrize("n", [1, 7, 256, 300])
@pytest.mark.parametrize("variant", VARIANTS)
def test_vit_batch_embeddings_match_oracle(tmp_path, variant, n):
    sd = _state(variant, 2)
    reid = _model(tmp_path, sd)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    boxes = _boxes(rng, n, 720, 1280)
    got = reid.get_features(boxes, img)
    _emb_ok(got, _DeviceOracle(sd, variant).get_features(boxes, img))
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    # a crop's row does not depend on its chunk or on its position in it (300 crops cross the 256-crop chunk)
    tail = slice(max(0, n - 5), n)
    assert np.array_equal(reid.get_features(boxes[tail], img), got[tail])


@pytest.mark.parametrize("kind", ["botsort", "deepocsort", "strongsort"])
def test_vit_trackers_match_oracle(tmp_path, kind):
    import boxmot_b200 as bb
    from oracle.streams import bench_stream

    sd = _state("vit_tiny_parts3", 5)
    reid = _model(tmp_path, sd)
    oracle_reid = _DeviceOracle(sd, "vit_tiny_parts3")
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


def test_create_tracker_with_vit_tiny_parts3_checkpoint(tmp_path):
    """A seeded checkpoint saved as the reference trainer saves it (`state_dict` with `module.` prefixes, classifiers,
    `model_name`) through create_tracker(reid_weights=...): converted once, 2048-d embeddings, tracks out."""
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream, make_vit_state

    sd = make_vit_state("vit_tiny_parts3", 4)
    pt = tmp_path / "vit_tiny_parts3_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_name": "vit_tiny_parts3"}, pt)
    trk = bb.create_tracker("botsort", reid_weights=pt, use_cmc=False)
    img, frames = bench_stream(24, 6, hw=(360, 640))
    n = sum(len(trk.update(d, img)) for d in frames)
    assert n > 0


def test_reference_abi_botsort_with_vit_model(tmp_path):
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(_state("vit_nano_ain_os", 6), tmp_path / "abi.b200reid")
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), b"resize", ctypes.byref(h)) == 1
    dim = ctypes.c_int(0)
    assert lib.boxmot_reid_capi_feature_dim(h, ctypes.byref(dim)) == 1 and dim.value == 192
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
