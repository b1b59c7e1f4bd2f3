"""MLFN on bench.py's default workload: the BoT-SORT tracker, detection stream and frame ring of BASELINE config 2 with
MLFN (seeded weights, 1024-d rows) as the ReID backbone, alternated in one process with ResNet50 on the same workload,
timed with bench.py's own device and end-to-end legs, plus parity of the first frames against the oracle tracker fed by
the oracle MLFN.  Prints one JSON line with frames/s, ReID device ms and crops per frame, the achieved TFLOP/s from
the algorithmic FLOP count of a crop, and the card's name and power limit read in the same call.

    python scripts/bench_mlfn.py [--steps 200] [--warmup 20] [--rounds 2] [--parity-frames 2]

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


def mlfn_gflop_per_crop(in_h=256, in_w=128):
    """Algorithmic GFLOP of one crop: 2 x MAC over every convolution of reid/backbones/mlfn.py (stem; per MLFNBlock
    fm_conv1, the grouped fm_conv2, fm_conv3, the downsample and the three FSM layers; fc_x and fc_s)."""
    from boxmot_b200.synthetic import MLFN_FEAT, MLFN_GROUPS, mlfn_blocks

    h, w = in_h // 2, in_w // 2
    macs = h * w * 64 * 3 * 49
    h, w = h // 2, w // 2
    for cin, cout, s, (f0, f1), ds in mlfn_blocks():
        mid = cout // 2
        ho, wo = h // s, w // s
        macs += h * w * cin * mid + ho * wo * 9 * (mid // MLFN_GROUPS) * mid + ho * wo * mid * cout
        macs += cin * f0 + f0 * f1 + f1 * MLFN_GROUPS + (ho * wo * cin * cout if ds else 0)
        h, w = ho, wo
    macs += 2048 * MLFN_FEAT + 16 * MLFN_GROUPS * MLFN_FEAT
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
    ap.add_argument("--rounds", type=int, default=2, help="alternations of MLFN and ResNet50")
    ap.add_argument("--parity-frames", type=int, default=2, help="first frames of stream 0 checked against the oracle (CPU)")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_mlfn.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    from boxmot_b200.synthetic import make_mlfn_state, make_resnet_state
    from boxmot_b200.weights import export_blob

    base = bench.CONFIGS[2]
    tmp = Path(tempfile.mkdtemp(prefix="b200mlfn_"))
    sd = make_mlfn_state(seed=0)
    models = {
        "mlfn": (dict(base, id=2, arch="mlfn", feat=1024), export_blob(sd, tmp / "mlfn_synthetic.b200reid")),
        "resnet50": (dict(base, id=2, arch="resnet50", feat=2048),
                     export_blob(make_resnet_state(50, seed=0), tmp / "resnet50_synthetic.b200reid")),
    }
    K, Wm = args.steps, max(3, args.warmup)
    runs = {name: [] for name in models}
    for _ in range(args.rounds):
        for name, (cfg, blob) in models.items():
            dev = bench.device_run(cfg, blob, K, Wm, None)
            e2e_ms, _, api = bench.e2e_run(cfg, blob, dev["per_stream"], K, Wm, None, pinned=False)
            reid_ms = sum(dev["prof"][c]["ms_per_step"] for c in bench.CLASSES if c != "association")
            runs[name].append(dict(dev=dev, e2e_ms=e2e_ms, api=api, reid_ms=reid_ms))

    cfg, blob = models["mlfn"]
    first = runs["mlfn"][0]["dev"]
    ps = first["per_stream"][0]
    from oracle.mlfn import get_features
    from oracle.trackers import BotSortOracle

    class OracleMlfn:
        def get_features(self, xyxys, img):
            return get_features(sd, xyxys, img)

    orc = BotSortOracle(reid_model=OracleMlfn(), **cfg["params"])
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

    gflop_crop = mlfn_gflop_per_crop()
    res = summary("mlfn")
    reid_ms = min(res["reid_device_ms_per_frame"])
    gflop_frame = res["crops_per_frame"] * gflop_crop
    achieved = gflop_frame / reid_ms   # GFLOP per ms = TFLOP/s
    line = {
        "metric": "tracker.update() frames/sec with MLFN ReID", "value": max(res["device_fps"]), "unit": "frames/s",
        "steps": K, "warmup": Wm, "rounds": args.rounds, "data": "synthetic",
        "workload": f"botsort workload of BASELINE config 2 ({base['dets']} dets/frame, {base['hw'][0]}x{base['hw'][1]}) "
                    f"with ReID in update(); mlfn and resnet50 alternated in one process",
        "card": power_limit(),
        "mlfn": res,
        "resnet50": summary("resnet50"),
        "roofline": {"kernel": "MLFN ReID (all kernels of a frame, serialised device time)",
                     "gflop_per_crop": gflop_crop, "algorithmic_gflop_per_frame": gflop_frame,
                     "achieved_tflops": achieved,
                     "fp32_floor_ms_per_frame": gflop_frame / FP32_PEAK_TFLOPS,
                     "peak_source": "H100 SXM data sheet (dense FP32 67 TFLOP/s, 700 W), not measured"},
        "parity": parity,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
