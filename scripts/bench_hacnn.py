"""HACNN on bench.py's default workload: the BoT-SORT tracker, detection stream and frame ring of BASELINE config 2 with
HACNN (seeded weights, 1024-d rows from 160x64 crops) as the ReID backbone, alternated in one process with the default
OSNet_x0_25 on the same workload, timed with bench.py's own device and end-to-end legs, plus parity of the first
frames against the oracle tracker fed by the oracle HACNN.  Prints one JSON line with frames/s, ReID device ms and crops per frame, the achieved TFLOP/s from
the algorithmic FLOP count of a crop, and the card's name and power limit read in the same call.

    python scripts/bench_hacnn.py [--steps 200] [--warmup 20] [--rounds 2] [--parity-frames 2]

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

FP32_PEAK_TFLOPS = 67.0    # H100 SXM data sheet, dense FP32 on the CUDA cores (700 W)


def hacnn_gflop_per_crop():
    """Algorithmic GFLOP of one crop as torch.utils.flop_counter counts reid/backbones/hacnn.py: 2 x MAC over every
    convolution and linear layer, the soft attention's C x C 1x1 over every pixel included (the kernels compute it as
    s[p] (W c)[o] + b[o]); pools, resizes and the STN are not counted."""
    from boxmot_b200.synthetic import hacnn_layout

    level = {1: (80, 32), 2: (40, 16), 3: (20, 8)}   # the Inception input map of each level
    local = {1: (24, 28), 2: (12, 14), 3: (6, 7)}    # the local branch's InceptionB input map
    macs = 0
    for name, kind, shape in hacnn_layout():
        if kind == "bn":
            continue
        if kind == "lin":
            macs += shape[0] * shape[1]
            continue
        co, ci, k = shape[0], shape[1], shape[2]
        if name == "conv":
            h, w = 80, 32
        elif name.startswith("ha"):
            fh, fw = level[int(name[2])]
            fh, fw = fh // 2, fw // 2   # the attended map
            h, w = (fh // 2, fw // 2) if name.endswith("conv1") and "spatial" in name else (fh, fw)
            if "channel_attn" in name:
                h, w = 1, 1
        else:
            ih, iw = local[int(name[10])] if name.startswith("local_conv") else level[int(name[9])]
            inc_b = name.startswith("local_conv") or name.split(".")[1] == "1"
            half = inc_b and name.endswith(("stream1.1", "stream2.2", "stream3.1"))
            h, w = ((ih - 1) // 2 + 1, (iw - 1) // 2 + 1) if half else (ih, iw)
            if name.startswith("local_conv"):
                h *= 4   # the four regions
        macs += h * w * co * ci * k * k
    return 2 * macs / 1e9


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of HACNN and OSNet_x0_25")
    ap.add_argument("--parity-frames", type=int, default=2, help="first frames of stream 0 checked against the oracle (CPU)")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_hacnn.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    from boxmot_b200.synthetic import make_hacnn_state, make_osnet_state
    from boxmot_b200.weights import export_blob

    base = bench.CONFIGS[2]
    tmp = Path(tempfile.mkdtemp(prefix="b200hacnn_"))
    sd = make_hacnn_state(seed=0)
    models = {
        "hacnn": (dict(base, id=2, arch="hacnn", feat=1024), export_blob(sd, tmp / "hacnn_synthetic.b200reid")),
        "osnet_x0_25": (base, export_blob(make_osnet_state("osnet_x0_25", seed=0), tmp / "osnet_x0_25.b200reid")),
    }
    K, Wm = args.steps, max(3, args.warmup)
    runs = {name: [] for name in models}
    for _ in range(args.rounds):
        for name, (cfg, blob) in models.items():
            dev = bench.device_run(cfg, blob, K, Wm, None)
            e2e_ms, _, api = bench.e2e_run(cfg, blob, dev["per_stream"], K, Wm, None, pinned=False)
            reid_ms = sum(dev["prof"][c]["ms_per_step"] for c in bench.CLASSES if c != "association")
            runs[name].append(dict(dev=dev, e2e_ms=e2e_ms, api=api, reid_ms=reid_ms))

    cfg, blob = models["hacnn"]
    first = runs["hacnn"][0]["dev"]
    ps = first["per_stream"][0]
    from oracle.hacnn import get_features
    from oracle.trackers import BotSortOracle

    class OracleHacnn:
        def get_features(self, xyxys, img):
            return get_features(sd, xyxys, img)

    orc = BotSortOracle(reid_model=OracleHacnn(), **cfg["params"])
    rows = [np.asarray(orc.update(ps[1][f], ps[0][f % cfg["ring"]]), np.float32).reshape(-1, 8)
            for f in range(args.parity_frames)]
    parity = bench.parity_check(cfg, blob, rows, first["per_stream"])

    def summary(name):
        rs = runs[name]
        best = min(rs, key=lambda r: r["dev"]["value_ms"])
        return {
            "device_fps": [K / (r["dev"]["value_ms"] * 1e-3) for r in rs],
            "e2e_fps": [K / (r["e2e_ms"] * 1e-3) for r in rs],
            "reid_device_ms_per_frame": [r["reid_ms"] for r in rs],
            "crops_per_frame": best["dev"]["crops"],
            "kernel_classes": best["dev"]["prof"],
        }

    gflop_crop = hacnn_gflop_per_crop()
    res = summary("hacnn")
    reid_ms = min(res["reid_device_ms_per_frame"])
    gflop_frame = res["crops_per_frame"] * gflop_crop
    achieved = gflop_frame / reid_ms   # GFLOP per ms = TFLOP/s
    line = {
        "metric": "tracker.update() frames/sec with HACNN ReID", "value": max(res["device_fps"]), "unit": "frames/s",
        "steps": K, "warmup": Wm, "rounds": args.rounds, "data": "synthetic",
        "workload": f"botsort workload of BASELINE config 2 ({base['dets']} dets/frame, {base['hw'][0]}x{base['hw'][1]}) "
                    f"with ReID in update(); hacnn and osnet_x0_25 alternated in one process",
        "card": power_limit(),
        "hacnn": res,
        "osnet_x0_25": summary("osnet_x0_25"),
        "roofline": {"kernel": "HACNN ReID (all kernels of a frame, serialised device time)",
                     "gflop_per_crop": gflop_crop, "algorithmic_gflop_per_frame": gflop_frame,
                     "achieved_tflops": achieved,
                     "fp32_floor_ms_per_frame": gflop_frame / FP32_PEAK_TFLOPS,
                     "peak_source": "H100 SXM data sheet (dense FP32 67 TFLOP/s, 700 W), not measured"},
        "parity": parity,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
