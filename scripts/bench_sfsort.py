"""SFSORT throughput on bench.py's default stream (256 detections per frame, 1280 x 720): device-resident frames/s with
S = 1, 16 and 256 streams per handle (`update_device` + one `fetch`), end-to-end frames/s through `SFSORT.update`, the CPU
oracle's time on the same stream, and an id-parity check of the timed frames against the oracle.  Prints one JSON line
with the GPU's name and power limit read in the same run.
    python scripts/bench_sfsort.py [--frames 60] [--warmup 10]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    import torch

    import boxmot_b200 as bb
    from boxmot_b200.synthetic import bench_stream
    from tests import sfsort_oracle

    img, frames = bench_stream(256, a.warmup + a.frames)
    hw = img.shape[:2]
    res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()}
    CD = 256
    for S in (1, 16, 256):
        m = bb.MultiStreamTracker("sfsort", n_streams=S, cap_tracks=512, cap_dets=CD)
        bufs = []
        for d in frames:
            b = np.zeros((S, CD, 6), np.float32)
            b[:, : len(d)] = d
            bufs.append(torch.from_numpy(b).cuda())
        rows = [len(d) for d in frames]
        for f in range(a.warmup):
            m.update_device(bufs[f], [rows[f]] * S, image_hw=hw, sync=False)
        m.fetch()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f in range(a.warmup, a.warmup + a.frames):
            m.update_device(bufs[f], [rows[f]] * S, image_hw=hw, sync=False)
        m.fetch()
        dt = time.perf_counter() - t0
        res[f"device_fps_S{S}"] = round(a.frames / dt, 1)
        res[f"device_stream_fps_S{S}"] = round(a.frames * S / dt, 1)
        m.close()
        del bufs
    t = bb.SFSORT(cap_tracks=512, cap_dets=CD)
    o = sfsort_oracle.make()
    gpu_rows, cpu_rows = [], []
    for f in range(a.warmup):
        t.update(frames[f], img)
    t0 = time.perf_counter()
    for f in range(a.warmup, a.warmup + a.frames):
        gpu_rows.append(t.update(frames[f], img))
    res["e2e_fps"] = round(a.frames / (time.perf_counter() - t0), 1)
    for f in range(a.warmup):
        o.update(frames[f], hw)
    t0 = time.perf_counter()
    for f in range(a.warmup, a.warmup + a.frames):
        cpu_rows.append(o.update(frames[f], hw))
    res["oracle_cpu_fps"] = round(a.frames / (time.perf_counter() - t0), 1)
    res["id_parity"] = all(np.array_equal(g, c) for g, c in zip(gpu_rows, cpu_rows))
    res["frames"], res["warmup"], res["dets_per_frame"] = a.frames, a.warmup, 256
    print(json.dumps(res))


if __name__ == "__main__":
    main()
