"""LMBN_n on a bench.py workload: the tracker, detection stream and frame ring of a BASELINE configuration with the
384x128 LMBN_n (seeded weights, 3584-d rows) as the ReID backbone, timed with bench.py's own device and end-to-end
legs, plus parity of the first frames against the oracle tracker fed by the oracle LMBN_n.  Prints one JSON line.

    python scripts/bench_lmbn.py [--config 2] [--steps 200] [--warmup 20] [--parity-frames 2]

Writes nothing into the tree (the blob goes to a temporary directory).  The LMBN_n kernels are float32 CUDA-core
kernels, so the share of peak is against the H100 SXM data sheet's dense FP32 rate."""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import bench  # noqa: E402

FP32_PEAK_TFLOPS = 67.0   # H100 SXM data sheet, dense FP32 on the CUDA cores (700 W)


def lmbn_n_gflop_per_crop(in_h=384, in_w=128):
    """Algorithmic GFLOP of one LMBN_n crop: 2 x MAC over every convolution of reid/backbones/lmbn/lmbn_n.py in eval
    (ChannelGate fc1 / fc2 and the 1x1 necks included, `shared` counted once per channel half)."""
    def osblock(hw, cin, cout):
        mid = cout // 4
        hid = mid // 16
        macs = hw * cin * mid + 10 * hw * (mid * mid + 9 * mid) + 4 * 2 * mid * hid + hw * mid * cout
        return macs + (hw * cin * cout if cin != cout else 0)

    h, w = in_h // 2, in_w // 2
    macs = h * w * 64 * 3 * 49                                   # stem 7x7/2
    hw = (h // 2) * (w // 2)                                     # after the max pool
    macs += osblock(hw, 64, 256) + osblock(hw, 256, 256) + hw * 256 * 256
    hw //= 4
    macs += osblock(hw, 256, 384)                                # trunk end
    branch = osblock(hw, 384, 384) + hw * 384 * 384
    hw //= 4
    branch += osblock(hw, 384, 512) + osblock(hw, 512, 512) + hw * 512 * 512
    macs += 3 * branch + osblock(hw, 512, 512)                   # three branches + the bottleneck
    macs += 5 * 512 * 512 + 2 * 256 * 512                        # reduction necks, `shared` on both halves
    return 2 * macs / 1e9


def oracle_tracker(cfg, sd):
    from oracle.lmbn import OracleReIDAny

    model = OracleReIDAny(sd)
    if cfg["kind"] == "botsort":
        from oracle.trackers import BotSortOracle

        return BotSortOracle(reid_model=model, **cfg["params"])
    if cfg["kind"] == "deepocsort":
        from oracle.deepocsort import DeepOcSortOracle

        return DeepOcSortOracle(reid_model=model, **cfg["params"])
    from oracle.strongsort import StrongSortOracle

    return StrongSortOracle(reid_model=model, **cfg["params"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2, choices=[2, 3, 4], help="BASELINE.json configuration whose workload runs")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--parity-frames", type=int, default=2, help="first frames of stream 0 checked against the oracle (CPU)")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_lmbn.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    from boxmot_b200.synthetic import make_lmbn_n_state
    from boxmot_b200.weights import export_blob

    base = bench.CONFIGS[args.config]
    cfg = dict(base, id=args.config, arch="lmbn_n", feat=3584,
               workload=f"{base['kind']} workload of BASELINE config {args.config} with LMBN_n (384x128) ReID in update(), "
                        f"{base['streams']} stream(s) x {base['dets']} dets/frame per GPU")
    K, Wm = args.steps, max(3, args.warmup)
    sd = make_lmbn_n_state(seed=0)
    blob = export_blob(sd, Path(tempfile.mkdtemp(prefix="b200lmbn_")) / "lmbn_n_synthetic.b200reid")

    dev = bench.device_run(cfg, blob, K, Wm, None)
    e2e_ms, _, api = bench.e2e_run(cfg, blob, dev["per_stream"], K, Wm, None, pinned=False)
    ps = dev["per_stream"][0]
    orc = oracle_tracker(cfg, sd)
    rows = [np.asarray(orc.update(ps[1][f], ps[0][f % cfg["ring"]]), np.float32).reshape(-1, 8)
            for f in range(args.parity_frames)]
    parity = bench.parity_check(cfg, blob, rows, dev["per_stream"])

    S, value_ms, prof = cfg["streams"], dev["value_ms"], dev["prof"]
    gflop_crop = lmbn_n_gflop_per_crop()
    gflop_step = dev["crops"] * gflop_crop
    achieved = gflop_step / (value_ms * 1e-3 / K) / 1e3   # TFLOP/s
    reid_ms = sum(prof[c]["ms_per_step"] for c in bench.CLASSES if c != "association")
    dom = max((c for c in bench.CLASSES if c != "association"), key=lambda c: prof[c]["ms_per_step"])
    line = {
        "metric": "tracker.update() frames/sec with LMBN_n ReID", "value": S * K / (value_ms * 1e-3), "unit": "frames/s",
        "steps": K, "warmup": Wm, "ms_per_step": value_ms / K, "dtype": "f32", "data": "synthetic",
        "config": {"workload": cfg["workload"], "baseline_config": args.config, "crops_per_step_per_gpu": dev["crops"],
                   "reid": "lmbn_n random-init (seed 0); float32 CUDA-core kernels"},
        "e2e": {"value": S * K / (e2e_ms * 1e-3), "unit": "frames/s", "ms_per_step": e2e_ms / K, "api": api},
        "device": torch.cuda.get_device_name(0),
        "clocks": dev["clocks"],
        "roofline": {"kernel": "ReID backbone (all conv kernels of a step)", "bound": "fp32", "achieved": achieved,
                     "peak": FP32_PEAK_TFLOPS, "unit": "TFLOP/s", "frac": achieved / FP32_PEAK_TFLOPS,
                     "peak_source": "H100 SXM data sheet (dense FP32, 700 W), not measured",
                     "gflop_per_crop": gflop_crop, "algorithmic_gflop_per_step": gflop_step,
                     "serialised_reid_ms_per_step": reid_ms, "dominant_class": dom,
                     "dominant_class_ms": prof[dom]["ms_per_step"]},
        "kernel_classes": prof,
        "parity": parity,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
