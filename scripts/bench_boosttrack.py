"""BoostTrack++ on the bench.py workload: BASELINE's default stream (1 x 256 detections/frame, 1280x720, the reference
generator) and the 16-stream line, with configs/trackers/boosttrack.yaml's parameters and OSNet_x0_25 (seeded weights) on
the device, timed with bench.py's device-resident leg (CUDA events) plus an end-to-end leg through
`BoostTrack.update(dets, img)`, and parity of the first frames against the oracle BoostTrack fed by the oracle ReID.
Camera-motion estimation is off, as in every bench.py configuration.  Prints one JSON line.

    python scripts/bench_boosttrack.py [--steps 200] [--warmup 20] [--parity-frames 2]

Writes nothing into the tree (the blob goes to a temporary directory)."""
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

import bench  # noqa: E402

PARAMS = {k: v for k, v in __import__("boxmot_b200.trackers", fromlist=["x"]).BOOSTTRACK_YAML_DEFAULTS.items()
          if k not in ("use_cmc", "cmc_method", "adaptive_kf")}


def gpu_power():
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
    ap.add_argument("--parity-frames", type=int, default=2)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_boosttrack.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    import boxmot_b200 as bb
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import make_osnet_state
    from boxmot_b200.weights import export_blob

    K, Wm = args.steps, max(3, args.warmup)
    sd = make_osnet_state("osnet_x0_25", seed=0)
    blob = export_blob(sd, Path(tempfile.mkdtemp(prefix="b200bt_")) / "osnet_x0_25_synthetic.b200reid")
    bench.n_crops = lambda cfg, d: len(d)   # BoostTrack embeds every detection row
    lines = {}
    for S in (1, 16):
        cfg = dict(bench.CONFIGS[2 if S == 1 else 5], kind="boosttrack", params=PARAMS,
                   workload=f"BoostTrack++ (boosttrack.yaml) + OSNet_x0_25 ReID in update(), {S} stream(s) x 256 dets/frame, "
                            "1280x720, CMC off")
        dev = bench.device_run(cfg, blob, K, Wm, None)
        ps = dev["per_stream"]
        lines[S] = dict(frames_per_s=S * K / (dev["value_ms"] * 1e-3), ms_per_step=dev["value_ms"] / K,
                        crops_per_step=dev["crops"], launches_per_step=dev["launches_per_step"],
                        reid_ms_per_step=sum(dev["prof"][c]["ms_per_step"] for c in bench.CLASSES if c != "association"),
                        association_ms_per_step=dev["prof"]["association"]["ms_per_step"])
        if S == 1:
            rows_above = float(np.mean([(ps[0][1][f][:, 4] >= PARAMS["det_thresh"]).sum() for f in range(Wm, Wm + K)]))
            lines[S]["rows_conf_above_det_thresh_before_boosts"] = rows_above
            trk = bb.BoostTrack(reid_model=B200ReID(blob), use_cmc=False, cap_tracks=1024, cap_dets=256, **PARAMS)
            for f in range(Wm):
                trk.update(ps[0][1][f], ps[0][0][f % cfg["ring"]])
            reid_ms, assoc_ms = [], []
            t0 = time.perf_counter()
            for f in range(Wm, Wm + K):
                trk.update(ps[0][1][f], ps[0][0][f % cfg["ring"]])
                a, b = trk._engine.last_device_ms()
                reid_ms.append(a)
                assoc_ms.append(b)
            e2e = 1e3 * (time.perf_counter() - t0)
            lines[S]["e2e"] = dict(frames_per_s=K / (e2e * 1e-3), ms_per_step=e2e / K, api="BoostTrack.update(dets, img)",
                                   last_device_ms_reid=float(np.mean(reid_ms)), last_device_ms_association=float(np.mean(assoc_ms)))
            from oracle import reid as orid
            from tests.boosttrack_oracle import BoostTrackOracle

            gpu = bb.BoostTrack(reid_model=B200ReID(blob), use_cmc=False, cap_tracks=1024, cap_dets=256, **PARAMS)
            orc = BoostTrackOracle(reid_model=orid.OracleReID(sd), **PARAMS)
            ok, n = True, 0
            for f in range(args.parity_frames):
                img = ps[0][0][f % cfg["ring"]]
                got = np.asarray(gpu.update(ps[0][1][f], img), np.float32)
                want = np.asarray(orc.update(ps[0][1][f], img), np.float32).reshape(-1, 8)
                n += len(want)
                ok = ok and got.shape == want.shape and np.array_equal(got[:, 4:], want[:, 4:])
            lines[S]["parity"] = dict(frames=args.parity_frames, rows=n, ids_conf_cls_det_ind_equal=bool(ok))
    print(json.dumps({"metric": "BoostTrack++ tracker.update() frames/sec at 256 dets/frame", "value": lines[1]["frames_per_s"],
                      "unit": "frames/s", "steps": K, "warmup": Wm, "device": torch.cuda.get_device_name(0),
                      "gpu_name_power_limit_max_sm_clock": gpu_power(), "one_stream": lines[1], "sixteen_streams": lines[16]}))


if __name__ == "__main__":
    main()
