"""Latency of the device SOF camera-motion estimator (boxmot_b200.SOF) against the reference's estimator on host OpenCV.

    python scripts/measure_sof.py [--frames N] [--warmup W]

For each frame size (720p, 1080p), one seeded camera_similarity_sequence is estimated frame by frame:
  * device: boxmot_b200.SOF.apply, host clock around each call (the call copies the BGR frame to the device and
    returns after a device synchronise, so it is the whole per-frame cost a caller pays);
  * host:   the same SOF.apply on the installed cv2 (tests/sof_oracle.py restates the reference's sof.py call for
    call), on this machine's CPU;
  * tracker: BoT-SORT without ReID (MultiStreamTracker.update, which returns after the device has finished) with
    set_cmc("sof") versus CMC off, at 1 and 16 streams (every stream gets the same sequence).  With CMC off the frames
    are not needed and not uploaded, so the difference includes the upload of the S frames.
Prints one JSON line with ms/frame (median and mean), the accept rate, and the GPU name and power limit.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, limit = [x.strip() for x in out[0].split(",")]
        return name, limit
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})", "unknown"


def time_calls(est, frames, dets, warmup):
    ts, accepted = [], 0
    for i, (im, d) in enumerate(zip(frames, dets)):
        t0 = time.perf_counter()
        est.apply(im, d)
        dt = (time.perf_counter() - t0) * 1e3
        if i >= warmup:
            ts.append(dt)
        accepted += getattr(est, "last_status", getattr(est, "status", None)) == 1
    return ts, accepted


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import boxmot_b200 as bb
    from boxmot_b200.synthetic import camera_similarity_sequence
    from tests.sof_oracle import SofOracle

    bb.require_device()
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit": limit, "frames": args.frames, "warmup": args.warmup, "sizes": {}}
    for hw in ((720, 1280), (1080, 1920)):
        frames, dets, _ = camera_similarity_sequence(args.frames, hw=hw, seed=71)
        dev_t, dev_acc = time_calls(bb.SOF(), frames, dets, args.warmup)
        host_t, host_acc = time_calls(SofOracle(), frames, dets, args.warmup)
        upd = {}
        for S in (1, 16):
            for cmc in (None, "sof"):
                trk = bb.MultiStreamTracker("botsort", n_streams=S, cap_tracks=256, cap_dets=64, feat_dim=512,
                                            with_reid=False)
                trk.set_cmc(cmc)
                ts = []
                for i, (im, d) in enumerate(zip(frames, dets)):
                    t0 = time.perf_counter()
                    trk.update([d] * S, [im] * S if cmc else None)
                    if i >= args.warmup:
                        ts.append((time.perf_counter() - t0) * 1e3)
                trk.close()
                upd[f"update_ms_S{S}_{cmc or 'off'}"] = round(statistics.median(ts), 3)
        res["sizes"][f"{hw[0]}p"] = {**upd,
            "device_ms_median": round(statistics.median(dev_t), 3), "device_ms_mean": round(statistics.mean(dev_t), 3),
            "host_cv2_ms_median": round(statistics.median(host_t), 3),
            "host_cv2_ms_mean": round(statistics.mean(host_t), 3),
            "device_accepted": dev_acc, "host_accepted": host_acc}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
