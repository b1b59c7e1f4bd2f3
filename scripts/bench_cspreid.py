"""CSPReID-n ReID throughput: seeded cspreid_n weights (1536-d rows), one frame with `--crops` boxes (default 256, one
chunk), `get_features` timed end to end (image upload, crop staging, the network, rows back to the host), alternated
round by round in one process with OSNet_x1_0 on the same frame.  Each timed call ends in a device synchronise (the rows
come back to the host).  Prints one JSON line: crops/s and ms per call for each model, the algorithmic GFLOP per crop
(torch.utils.flop_counter over the float64 oracle, 2 x MAC of every convolution and GEMV) with the achieved TFLOP/s,
the max deviation of the first rows from the float64 oracle, and the card's name and power limit read in the same call.

    python scripts/bench_cspreid.py [--crops 256] [--steps 50] [--warmup 10] [--rounds 3] [--hw 256x128]

Writes nothing into the tree (the checkpoints go to a temporary directory)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def gflop_per_crop(hw):
    import torch
    from torch.utils.flop_counter import FlopCounterMode

    from boxmot_b200.synthetic import make_cspreid_state
    from tests import cspreid_oracle as oc

    sd = oc.double_state(make_cspreid_state(0))
    with FlopCounterMode(display=False) as fc:
        oc.forward_taps(sd, torch.zeros(1, 3, *hw, dtype=torch.float64))
    return fc.get_total_flops() / 1e9


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--crops", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hw", default="256x128", choices=["256x128", "256x256"])
    args = ap.parse_args()

    import torch

    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import make_cspreid_state, make_osnet_state
    from tests import cspreid_oracle as oc
    from tests import vit_oracle as ov

    hw = (256, 128) if args.hw == "256x128" else (256, 256)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 255, size=(720, 1280, 3), dtype=np.uint8)
    cx, cy = rng.uniform(0, 1280, args.crops), rng.uniform(0, 720, args.crops)
    bw, bh = rng.uniform(20, 120, args.crops), rng.uniform(40, 240, args.crops)
    boxes = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)
    sd = make_cspreid_state(1)
    with tempfile.TemporaryDirectory() as d:
        pt = Path(d) / ("cspreid_n_market1501.pt" if hw[1] == 128 else "cspreid_n_veri.pt")
        torch.save({"state_dict": sd}, pt)
        osnet = Path(d) / "osnet_x1_0_market1501.pt"
        torch.save(make_osnet_state("osnet_x1_0", 1), osnet)
        models = {"cspreid_n": B200ReID(pt), "osnet_x1_0": B200ReID(osnet)}
    assert models["cspreid_n"].input_shape == hw

    # parity of the first rows against the float64 oracle
    k = min(16, args.crops)
    x = ov.get_crops(boxes[:k], img, "resize", hw)
    want = oc.embed(oc.double_state(sd), x.double()).numpy()
    got = models["cspreid_n"].get_features(boxes[:k], img)
    parity = float(np.abs(got - want).max())

    for m in models.values():
        for _ in range(args.warmup):
            m.get_features(boxes, img)
    times = {name: [] for name in models}
    for _ in range(args.rounds):
        for name, m in models.items():
            t0 = time.perf_counter()
            for _ in range(args.steps):
                m.get_features(boxes, img)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / args.steps)
    gf = gflop_per_crop(hw)
    out = {"crops": args.crops, "hw": list(hw), "steps": args.steps, "rounds": args.rounds, "card": card(),
           "gflop_per_crop": round(gf, 4), "max_abs_dev_vs_float64": parity}
    for name, ts in times.items():
        best, med = min(ts), float(np.median(ts))
        out[name] = {"ms_per_call_best": round(best * 1e3, 3), "ms_per_call_median": round(med * 1e3, 3),
                     "ms_per_call_rounds": [round(t * 1e3, 3) for t in ts],
                     "crops_per_s": round(args.crops / best, 1)}
    out["cspreid_n"]["tflops_achieved"] = round(gf * args.crops / min(times["cspreid_n"]) / 1e3, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
