#!/usr/bin/env python
"""reid_fingerprint.py -- bit-level fingerprint of every ReID backbone and kernel switch, for comparing two builds.

    python scripts/reid_fingerprint.py OUT.json

For each model, built from the seeded `boxmot_b200.synthetic` states and exported with `export_blob`, it records:
  - the SHA-256 of `get_features` on a seeded image with 300 boxes (more than one chunk);
  - the SHA-256 and floats per crop of every debug tap up to the first "stage index out of range" (and of tap 50, the
    fused crop of the tensor-core OSNet path), and the index where the taps end;
  - for a BoT-SORT tracker running that model for a few frames, `last_launches()` and the per-class launch counts of
    the tracker profile.
Only public APIs are used, so the same file runs against an older checkout; two builds that compute the same thing
write identical files.  Needs a CUDA device.
"""
from __future__ import annotations

import ctypes
import hashlib
import json
import os
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402

SWITCHES = ["BOXMOT_B200_REID_FP32", "BOXMOT_B200_REID_CHUNK", "BOXMOT_B200_REID_TC", "BOXMOT_B200_LIGHT_CHAIN",
            "BOXMOT_B200_CHAIN_VAR", "BOXMOT_B200_LIGHT_V1", "BOXMOT_B200_PW_V1", "BOXMOT_B200_LIGHT_TC",
            "BOXMOT_B200_LIGHT_SMALL", "BOXMOT_B200_PW_SMALL"]
# the switch sets of tests/test_gpu_reid.py::test_alternative_kernel_paths_keep_parity (which starts from FP32=1)
ALT_ENVS = [{"BOXMOT_B200_REID_FP32": "0", "BOXMOT_B200_REID_CHUNK": "32"},
            {"BOXMOT_B200_REID_FP32": "0", "BOXMOT_B200_REID_CHUNK": "24"}, {},
            {"BOXMOT_B200_REID_TC": "1"}, {"BOXMOT_B200_REID_CHUNK": "32"},
            {"BOXMOT_B200_REID_CHUNK": "256", "BOXMOT_B200_REID_TC": "1"},
            {"BOXMOT_B200_LIGHT_CHAIN": "0"}, {"BOXMOT_B200_CHAIN_VAR": "0"},
            {"BOXMOT_B200_CHAIN_VAR": "1", "BOXMOT_B200_REID_CHUNK": "24"},
            {"BOXMOT_B200_LIGHT_V1": "1"}, {"BOXMOT_B200_PW_V1": "1"},
            {"BOXMOT_B200_LIGHT_TC": "1"}, {"BOXMOT_B200_LIGHT_SMALL": "1"},
            {"BOXMOT_B200_PW_SMALL": "0"}]
BOTSORT = dict(track_high_thresh=0.6, new_track_thresh=0.62, appearance_thresh=0.6, proximity_thresh=0.6)
N_CLASSES = 9   # reid kernel classes + association, as bench.py reads them


def _models():
    from boxmot_b200 import synthetic as syn

    yield "osnet_x0_25", lambda: syn.make_osnet_state("osnet_x0_25", seed=7), {}
    yield "osnet_x0_25_fp32", lambda: syn.make_osnet_state("osnet_x0_25", seed=7), {"BOXMOT_B200_REID_FP32": "1"}
    yield "osnet_x1_0", lambda: syn.make_osnet_state("osnet_x1_0", seed=3), {}
    yield "mobilenetv2_x1_4", lambda: syn.make_mobilenetv2_state(1.4, seed=6), {}
    yield "lmbn_n", lambda: syn.make_lmbn_n_state(seed=4), {}
    yield "osnet_ain_x0_25", lambda: syn.make_osnet_ain_state("x0_25", seed=5), {}
    yield "osnet_ibn_x1_0", lambda: syn.make_osnet_ibn_state(seed=8), {}
    yield "resnet50", lambda: syn.make_resnet_state(50, seed=2), {}
    yield "clip", lambda: syn.make_clip_state(2), {}
    yield "clip_vehicle", lambda: syn.make_clip_state(3, vehicle=True), {}
    for i, env in enumerate(ALT_ENVS):
        yield f"osnet_x0_25_alt{i}", lambda: syn.make_osnet_state("osnet_x0_25", seed=9), \
            {"BOXMOT_B200_REID_FP32": "1", **env}


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _boxes(rng, n, hw):
    h, w = hw
    cx, cy = rng.uniform(0, w, n), rng.uniform(0, h, n)
    bw, bh = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    return np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)


def fingerprint(blob) -> dict:
    import torch

    import boxmot_b200 as bb
    from boxmot_b200 import _lib
    from boxmot_b200.reid import B200Error, B200ReID
    from boxmot_b200.synthetic import bench_stream

    rng = np.random.default_rng(1)
    img = rng.integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    reid = B200ReID(blob)
    out = {"features": _sha(reid.get_features(_boxes(rng, 300, img.shape[:2]), img))}
    tap_boxes = _boxes(rng, 20, img.shape[:2])   # a tap holds one chunk of crops, and the smallest chunk here is 24
    taps = []
    for stage in range(100):
        try:
            t = reid.debug_stage(tap_boxes, img, stage)
        except B200Error as e:
            assert "stage index out of range" in str(e), e
            break
        taps.append([t.shape[1], _sha(t)])
    out["taps"], out["taps_end"] = taps, len(taps)
    try:   # the fused crop of the tensor-core OSNet path
        t = reid.debug_stage(tap_boxes, img, 50)
        out["tap50"] = [t.shape[1], _sha(t)]
    except B200Error as e:
        out["tap50"] = str(e)
    feat = reid.feature_dim
    reid.close()

    lib = _lib.require_device()
    trk = bb.MultiStreamTracker("botsort", n_streams=1, cap_tracks=256, cap_dets=64, feat_dim=feat,
                                reid_blob=str(blob), **BOTSORT)
    frame, dets = bench_stream(64, 6, hw=(360, 640))
    d_img = torch.from_numpy(frame).cuda()
    d_dets = torch.from_numpy(np.stack(dets)[:, None].astype(np.float32)).cuda().contiguous()
    rows = (ctypes.c_int * 1)(64)

    def step(f):
        ok = lib.boxmot_b200_tracker_update_device(trk.handle, d_dets[f].data_ptr(), rows, None, d_img.data_ptr(),
                                                   360, 640, 1)
        assert ok, _lib.last_error(lib)

    for f in range(4):
        step(f)
    out["last_launches"] = trk.last_launches()
    lib.boxmot_b200_tracker_profile(trk.handle, 1)
    step(4)
    step(5)
    cls_ms = (ctypes.c_double * N_CLASSES)()
    cls_n = (ctypes.c_int * N_CLASSES)()
    lib.boxmot_b200_tracker_profile_read(trk.handle, cls_ms, cls_n)
    lib.boxmot_b200_tracker_profile(trk.handle, 0)
    out["profile_launches"] = list(cls_n)
    trk.close()
    return out


def main():
    result = {}
    with tempfile.TemporaryDirectory() as tmp:
        from boxmot_b200.weights import export_blob

        for name, make, env in _models():
            for k in SWITCHES:
                os.environ.pop(k, None)
            os.environ.update(env)
            blob = export_blob(make(), Path(tmp) / f"{name}.b200reid")
            result[name] = fingerprint(blob)
            print(name, result[name]["features"][:16], result[name].get("taps_end"), result[name]["last_launches"],
                  flush=True)
    Path(sys.argv[1]).write_text(json.dumps(result, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
