"""OSNet-AIN on the default bench.py workload: BoT-SORT with 256 detections per frame (BASELINE config 2's tracker,
detection stream and frame ring) with osnet_ain_x1_0 as the ReID backbone, alternated in one process with osnet_x1_0
(three runs each, seeded weights), timed with bench.py's own device-resident and end-to-end legs.  A separate
torch.profiler run over B200ReID times the instance-norm kernels (k_in_stats, k_in_apply, k_maxpool3s2_in) and reports
their achieved bytes/s, with the bytes computed from the layer shapes, against the H100 SXM's 3.35 TB/s HBM3.
Prints one JSON line.

    python scripts/bench_osnet_in.py [--steps 100] [--warmup 10] [--runs 3]

Writes nothing into the tree (the blobs go to a temporary directory)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import bench  # noqa: E402

HBM_TBS = 3.35   # H100 SXM data sheet HBM3 bandwidth, not measured
IN_KERNELS = ("k_in_stats", "k_in_apply", "k_maxpool3s2_in")


def in_bytes_per_crop(c=(64, 256, 384, 512)):
    """HBM bytes the instance-norm kernels of one osnet_ain_x1_0 crop move at least once (float32): the stem's statistics
    read the 128x64xc0 map, its fused pool reads it again and writes the 64x32xc0 map; each OSBlockINin (conv2.0, conv2.1,
    conv3.1, conv4.0) reads conv3's map for the statistics, then reads it and the identity and writes the output."""
    stem = 128 * 64 * c[0]
    total = 2 * stem + stem // 4
    for hw, ch in ((64 * 32, c[1]), (64 * 32, c[1]), (32 * 16, c[2]), (16 * 8, c[3])):
        total += 4 * hw * ch
    return 4 * total


def card():
    """Card name and power limit, read in one nvidia-smi query (read-only)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit_w": float(limit)}
    except Exception as e:   # noqa: BLE001
        return {"name": None, "power_limit_w": None, "error": str(e)}


def profile_in_kernels(blob, n_crops=256, reps=5):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import bench_stream

    reid = B200ReID(blob)
    img, frames = bench_stream(n_crops, 1)
    boxes = frames[0][:, :4]
    reid.get_features(boxes, img)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            reid.get_features(boxes, img)
        torch.cuda.synchronize()
    us = {k: 0.0 for k in IN_KERNELS}
    total_us = 0.0
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        total_us += ev.device_time
        for k in IN_KERNELS:
            if k in ev.name:
                us[k] += ev.device_time
    reid.close()
    in_s = sum(us.values()) * 1e-6 / reps
    nbytes = in_bytes_per_crop() * n_crops
    return {"crops": n_crops, "reps": reps, "in_kernel_us_per_call": {k: v / reps for k, v in us.items()},
            "in_share_of_reid_device_time": sum(us.values()) / total_us if total_us else None,
            "in_bytes_per_call": nbytes, "in_achieved_tbs": nbytes / in_s / 1e12 if in_s else None,
            "in_frac_of_hbm": (nbytes / in_s / 1e12) / HBM_TBS if in_s else None,
            "hbm_peak_tbs": HBM_TBS, "hbm_peak_source": "H100 SXM data sheet, not measured"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_osnet_in.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    from boxmot_b200.synthetic import make_osnet_ain_state, make_osnet_state
    from boxmot_b200.weights import export_blob

    tmp = Path(tempfile.mkdtemp(prefix="b200osnet_in_"))
    blobs = {"osnet_x1_0": export_blob(make_osnet_state("osnet_x1_0", seed=0), tmp / "osnet_x1_0.b200reid"),
             "osnet_ain_x1_0": export_blob(make_osnet_ain_state("x1_0", 0), tmp / "osnet_ain_x1_0.b200reid")}
    K, Wm = args.steps, max(3, args.warmup)
    runs = {name: {"device_fps": [], "e2e_fps": []} for name in blobs}
    clocks = None
    for _ in range(args.runs):
        for name, blob in blobs.items():
            cfg = dict(bench.CONFIGS[2], id=2, arch=name)
            dev = bench.device_run(cfg, blob, K, Wm, None, profile=False)
            e2e_ms, _, _ = bench.e2e_run(cfg, blob, dev["per_stream"], K, Wm, None, pinned=False)
            runs[name]["device_fps"].append(cfg["streams"] * K / (dev["value_ms"] * 1e-3))
            runs[name]["e2e_fps"].append(cfg["streams"] * K / (e2e_ms * 1e-3))
            clocks = dev["clocks"]
    summary = {name: {k + "_median": float(np.median(v)) for k, v in r.items()} | r for name, r in runs.items()}
    line = {
        "metric": "BoT-SORT frames/s with osnet_ain_x1_0 vs osnet_x1_0 ReID (256 dets/frame, 1280x720)",
        "unit": "frames/s", "steps": K, "warmup": Wm, "runs": args.runs, "alternated": True,
        "results": summary,
        "ain_over_osnet_device": summary["osnet_ain_x1_0"]["device_fps_median"] / summary["osnet_x1_0"]["device_fps_median"],
        "instance_norm_kernels": profile_in_kernels(blobs["osnet_ain_x1_0"]),
        "card": card(), "clocks_last_run": clocks,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
