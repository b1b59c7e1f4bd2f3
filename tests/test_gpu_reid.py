"""GPU ReID parity through the C ABI: staged crops bit-exact, every stage of OSNet against the oracle, final
embeddings against the golden dumped from the reference classes and against the oracle at batch size, and
BoT-SORT with on-device ReID against the oracle tracker fed by the oracle ReID.
Embedding tolerance (BASELINE.json: 1e-4 rel): max |delta| <= 1e-4 * ||e||_inf per row (SURVEY H2: 46% of the
outputs are exact zeros, so an elementwise relative bound is ill-defined)."""
import hashlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import reid as orid
from tests.common import BOTSORT_YAML, GOLDEN

STAGES = {1: "stem", 2: "pool", 3: "conv2.0", 4: "conv2.1", 5: "conv2.2", 6: "conv3.0", 7: "conv3.1", 8: "conv3.2",
          9: "conv4.0", 10: "conv4.1"}


def _model(tmp_path, arch="osnet_x0_25", seed=7):
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.weights import export_blob

    sd = orid.make_osnet_state(arch, seed=seed)
    blob = export_blob(sd, tmp_path / f"{arch}_{seed}.b200reid")
    return sd, B200ReID(blob)


def _emb_ok(got, want):
    err = np.abs(got - want).max(axis=1)
    bound = 1e-4 * np.abs(want).max(axis=1)
    assert (err <= bound).all(), f"embedding error {err.max():.3e} exceeds 1e-4*||e||inf ({bound.min():.3e})"
    return float((err / np.abs(want).max(axis=1)).max())


def test_crops_bit_exact_and_golden(tmp_path):
    z = np.load(GOLDEN / "reid_osnet_x0_25.npz")
    sd, reid = _model(tmp_path, seed=int(z["weight_seed"]))
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    blob = reid.debug_stage(z["boxes"], img, 0).reshape(-1, 256, 128, 3)
    nchw = np.ascontiguousarray(blob.transpose(0, 3, 1, 2))
    assert np.array_equal(nchw[z["crops_sample_index"]], z["crops_sample"])
    assert hashlib.sha256(nchw.tobytes()).hexdigest() == str(z["crops_sha256"]), "crop staging must be bit-exact"
    # the product path stages crops inside the fused tensor-core front kernel: its resized uint8 values (tap 50) must be
    # the reference's too (RGB order, before the float conversion)
    fused = reid.debug_stage(z["boxes"], img, 50).reshape(-1, 256, 128, 3)
    assert np.array_equal(fused, orid.crop_boxes(z["boxes"], img).astype(np.float32)), "fused crop staging must be bit-exact"
    feats = reid.get_features(z["boxes"], img)
    rel = _emb_ok(feats, z["features"])
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-5
    cos = (feats * z["features"]).sum(1)
    assert cos.min() > 0.999999  # the reference's own cross-stack bar is cosine > 0.99 (tests/unit/test_reid_capi.py:165)
    print("max rel-to-inf-norm embedding error", rel)


def test_every_stage_matches_oracle(tmp_path):
    sd, reid = _model(tmp_path, seed=11)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 255, size=(360, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 380, 330], [-20, -10, 60, 100], [600, 300, 700, 400],
                      [100.5, 50.5, 101.4, 52.2]], np.float32)
    _, want = orid.osnet_forward(sd, orid.get_crops(boxes, img), return_stages=True)
    for idx, name in STAGES.items():
        w = want[name].permute(0, 2, 3, 1).contiguous().numpy().reshape(len(boxes), -1)
        g = reid.debug_stage(boxes, img, idx)
        assert g.shape == w.shape, (name, g.shape, w.shape)
        # the stem tap (1) is the float32 kernel; pool (2, fused front kernel) and the blocks run on the tensor cores with split-BF16 operands (a few 1e-6 of the
        # output scale per GEMM): 5e-5 of the stage's scale, the embedding bound itself stays 1e-4
        tol = (2e-5 if idx < 2 else 5e-5) * max(1.0, float(np.abs(w).max()))
        assert np.abs(g - w).max() < tol, f"stage {name}: max err {np.abs(g - w).max():.3e}"


@pytest.mark.parametrize("arch,n", [("osnet_x0_25", 256), ("osnet_x0_25", 131), ("osnet_x1_0", 24)])
def test_batch_embeddings_match_oracle(tmp_path, arch, n):
    sd, reid = _model(tmp_path, arch=arch, seed=2)
    rng = np.random.default_rng(n)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    cx, cy = rng.uniform(0, 1280, n), rng.uniform(0, 720, n)
    w, h = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    boxes = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1).astype(np.float32)
    got = reid.get_features(boxes, img)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    want = orid.get_features(sd, boxes, img)
    _emb_ok(got, want)
    # staged quartet == one-call path
    st = reid.inference_postprocess(reid.forward(reid.inference_preprocess(reid.get_crops(boxes, img))))
    assert np.array_equal(st, got)
    assert reid.get_features(np.zeros((0, 4), np.float32), img).size == 0


def test_botsort_with_device_reid_matches_oracle(tmp_path):
    import boxmot_b200 as bb
    from oracle.streams import bench_stream
    from oracle.trackers import BotSortOracle
    from tests.common import assert_rows_match

    sd, reid = _model(tmp_path, seed=5)
    img, frames = bench_stream(48, 12, hw=(360, 640))
    orc = BotSortOracle(reid_model=orid.OracleReID(sd), **BOTSORT_YAML)
    gpu = bb.BotSort(reid_model=reid, cap_tracks=256, cap_dets=128, **BOTSORT_YAML)
    assert gpu.provides_reid
    for f, d in enumerate(frames):
        assert_rows_match(gpu.update(d, img), orc.update(d, img), f)


def test_reid_abi_errors(tmp_path):
    import ctypes

    from boxmot_b200 import _lib

    lib = _lib.require_device()
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(b"/nonexistent.b200reid", None, ctypes.byref(h)) == 0
    assert b"cannot open" in lib.boxmot_reid_capi_last_error()
    bad = tmp_path / "bad.b200reid"
    bad.write_bytes(b"\x00" * 128)
    assert lib.boxmot_reid_capi_create(str(bad).encode(), None, ctypes.byref(h)) == 0
    sd, reid = _model(tmp_path)
    out = np.empty((1, 512), np.float32)
    img = np.zeros((32, 32, 4), np.uint8)
    box = np.array([[0, 0, 10, 10]], np.float32)
    assert lib.boxmot_reid_capi_compute_features(reid.handle, box.ctypes.data, 1, img.ctypes.data, 32, 32, 4,
                                                 out.ctypes.data, 512) == 0
    assert lib.boxmot_reid_capi_postprocess(reid.handle, out.ctypes.data, 512) == 0  # nothing staged


@pytest.mark.parametrize("env", [{"BOXMOT_B200_REID_FP32": "0", "BOXMOT_B200_REID_CHUNK": "32"},
                                 {"BOXMOT_B200_REID_FP32": "0", "BOXMOT_B200_REID_CHUNK": "24"}, {},
                                 {"BOXMOT_B200_REID_TC": "1"}, {"BOXMOT_B200_REID_CHUNK": "32"},
                                 {"BOXMOT_B200_REID_CHUNK": "256", "BOXMOT_B200_REID_TC": "1"},
                                 {"BOXMOT_B200_LIGHT_CHAIN": "0"}, {"BOXMOT_B200_CHAIN_VAR": "0"},
                                 {"BOXMOT_B200_CHAIN_VAR": "1", "BOXMOT_B200_REID_CHUNK": "24"},
                                 {"BOXMOT_B200_LIGHT_V1": "1"}, {"BOXMOT_B200_PW_V1": "1"},
                                 {"BOXMOT_B200_LIGHT_TC": "1"}, {"BOXMOT_B200_LIGHT_SMALL": "1"},
                                 {"BOXMOT_B200_PW_SMALL": "0"}])
def test_alternative_kernel_paths_keep_parity(tmp_path, monkeypatch, env):
    """Every selectable kernel generation / configuration keeps the embeddings within the bound: tensor-core (tf32 x3)
    pointwise path, other chunk sizes, per-level vs whole-branch LightConv, first-generation kernels."""
    # the tensor-core path (wgmma + TMA) is the default; every other switch selects among the float32 kernels
    monkeypatch.setenv("BOXMOT_B200_REID_FP32", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sd, reid = _model(tmp_path, seed=9)
    rng = np.random.default_rng(3)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    n = 70
    cx, cy = rng.uniform(0, 640, n), rng.uniform(0, 480, n)
    w, h = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    boxes = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1).astype(np.float32)
    _emb_ok(reid.get_features(boxes, img), orid.get_features(sd, boxes, img))


def test_mobilenetv2_x1_4_embeddings_match_oracle(tmp_path):
    """Row a4: MobileNetV2_x1_4 (1792-d), channel counts 22/33/89/134 padded to multiples of 4."""
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import make_mobilenetv2_state
    from boxmot_b200.weights import export_blob

    sd = make_mobilenetv2_state(1.4, seed=6)
    reid = B200ReID(export_blob(sd, tmp_path / "mobilenetv2_x1_4.b200reid"))
    assert reid.feature_dim == 1792
    rng = np.random.default_rng(4)
    img = rng.integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    n = 70
    cx, cy = rng.uniform(0, 960, n), rng.uniform(0, 540, n)
    w, h = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    boxes = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1).astype(np.float32)
    got = reid.get_features(boxes, img)
    want = orid.get_features(sd, boxes, img)
    assert got.shape == (n, 1792)
    _emb_ok(got, want)


@pytest.mark.parametrize("kind,kw", [
    ("botsort", dict(track_high_thresh=0.6, new_track_thresh=0.62, appearance_thresh=0.6, proximity_thresh=0.6)),
    ("deepocsort", dict(det_thresh=0.3)),
    ("strongsort", dict(min_conf=0.3, max_cos_dist=0.4, n_init=2))])
def test_pipelined_device_path_equals_synchronous(tmp_path, kind, kw):
    """update_device without per-frame sync overlaps ReID(f+1) with association(f) on two CUDA streams (every tracker
    family with on-device ReID); the tracker state after N frames must be identical to the frame-by-frame synchronous
    run."""
    import ctypes

    import torch

    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream, make_osnet_state
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(make_osnet_state("osnet_x0_25", seed=3), tmp_path / "pipe.b200reid")
    img, dets = bench_stream(48, 24, hw=(360, 640))
    imgs = np.stack([np.roll(img, 7 * k, axis=1) for k in range(4)])
    d_imgs = torch.from_numpy(imgs).cuda()
    d_dets = torch.from_numpy(np.stack(dets)[:, None].astype(np.float32)).cuda().contiguous()
    rows = (ctypes.c_int * 1)(48)
    snaps = []
    for sync in (1, 0):
        trk = bb.MultiStreamTracker(kind, n_streams=1, cap_tracks=256, cap_dets=48, feat_dim=512,
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


@pytest.mark.parametrize("n_dets", [5, 70])
def test_pipelined_multistream_with_empty_frames(tmp_path, n_dets):
    """Two streams in one handle, frames where a stream has no detections, crop counts below and above the slicing
    threshold: the pipelined device path (ReID slices on helper streams, association on the main stream) must leave
    exactly the state of the synchronous path."""
    import ctypes

    import torch

    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.synthetic import bench_stream, make_osnet_state
    from boxmot_b200.weights import export_blob

    lib = _lib.require_device()
    blob = export_blob(make_osnet_state("osnet_x0_25", seed=5), tmp_path / "pipe2.b200reid")
    S, F, CD = 2, 16, 80
    img, d0 = bench_stream(n_dets, F, hw=(360, 640))
    _, d1 = bench_stream(n_dets, F, hw=(360, 640), stream=1)
    imgs = torch.from_numpy(np.stack([img, np.roll(img, 11, axis=0)])).cuda()          # one frame per stream
    dets = np.zeros((F, S, CD, 6), np.float32)
    counts = np.zeros((F, S), np.int32)
    for f in range(F):
        for si, d in enumerate((d0[f], d1[f])):
            n = 0 if (f % 5 == 2 and si == 1) or f == 7 else len(d)       # empty stream / entirely empty frame
            dets[f, si, :n] = d[:n]
            counts[f, si] = n
    d_dets = torch.from_numpy(dets).cuda().contiguous()
    kw = dict(track_high_thresh=0.6, new_track_thresh=0.62, appearance_thresh=0.6, proximity_thresh=0.6)
    results = []
    for sync in (1, 0):
        trk = bb.MultiStreamTracker("botsort", n_streams=S, cap_tracks=256, cap_dets=CD, feat_dim=512,
                                    reid_blob=str(blob), **kw)
        for f in range(F):
            rows = (ctypes.c_int * S)(*counts[f].tolist())
            ok = lib.boxmot_b200_tracker_update_device(trk.handle, d_dets[f].data_ptr(), rows, None,
                                                       imgs.data_ptr(), 360, 640, sync)
            assert ok, _lib.last_error(lib)
        outs = [np.zeros((CD, 9), np.float32) for _ in range(S)]
        o_ptr = (ctypes.c_void_p * S)(*[o.ctypes.data for o in outs])
        o_cap = (ctypes.c_int * S)(*[CD] * S)
        o_rows = (ctypes.c_int * S)()
        assert lib.boxmot_b200_tracker_fetch(trk.handle, o_ptr, o_cap, o_rows), _lib.last_error(lib)
        results.append(([outs[i][: o_rows[i]].copy() for i in range(S)], [trk.snapshot(i) for i in range(S)]))
        trk.close()
    (rows_a, st_a), (rows_b, st_b) = results
    for i in range(S):
        assert np.array_equal(rows_a[i], rows_b[i])
        assert sorted(st_a[i]) == sorted(st_b[i]) and len(st_a[i]) > 0
        for k in st_a[i]:
            assert np.array_equal(st_a[i][k][0], st_b[i][k][0]) and np.array_equal(st_a[i][k][1], st_b[i][k][1])


def test_resize_pad_preprocess_matches_oracle(tmp_path):
    """preprocess="resize_pad" (reid/core/preprocessing.py:21-45; what a NULL preprocess name means in the reference's
    native ABI): staged crops bit-exact on both device paths (fused tensor-core front kernel, float32 staging kernel),
    embeddings within the bound, and NULL on the C ABI selects it."""
    import ctypes

    from boxmot_b200 import _lib
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.weights import export_blob

    sd = orid.make_osnet_state("osnet_x0_25", seed=13)
    blob = export_blob(sd, tmp_path / "pad.b200reid")
    reid = B200ReID(blob, preprocess="resize_pad")
    rng = np.random.default_rng(17)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = np.array([[10, 20, 90, 200], [300, 100, 460, 180], [-20, -10, 60, 100], [600, 300, 700, 400], [5, 5, 300, 470],
                      [100.5, 50.5, 101.4, 52.2], [200, 100, 230, 330]], np.float32)
    want_u8 = orid.crop_boxes(boxes, img, "resize_pad").astype(np.float32)
    assert np.array_equal(reid.debug_stage(boxes, img, 50).reshape(-1, 256, 128, 3), want_u8)
    blob0 = reid.debug_stage(boxes, img, 0).reshape(-1, 256, 128, 3)
    assert np.array_equal(blob0, orid.get_crops(boxes, img, "resize_pad").permute(0, 2, 3, 1).numpy())
    _emb_ok(reid.get_features(boxes, img), orid.get_features(sd, boxes, img, "resize_pad"))
    assert np.abs(reid.get_features(boxes, img) - B200ReID(blob).get_features(boxes, img)).max() > 1e-3   # it is a different staging
    # the reference's native ABI: NULL preprocess == "resize_pad" (base/src/reid_capi.cpp:83)
    lib = _lib.require_device()
    h = ctypes.c_void_p()
    assert lib.boxmot_reid_capi_create(str(blob).encode(), None, ctypes.byref(h)) == 1
    out = np.empty((len(boxes), 512), np.float32)
    assert lib.boxmot_reid_capi_compute_features(h, boxes.ctypes.data, len(boxes), img.ctypes.data, 480, 640, 3, out.ctypes.data, out.size) == 1
    assert np.array_equal(out, reid.get_features(boxes, img))
    lib.boxmot_reid_capi_destroy(h)
    with pytest.raises(ValueError):
        B200ReID(blob, preprocess="letterbox")
