"""OccluBoost next to BoostTrack++ on the bench.py workload: BASELINE's default stream (1 x 256 detections/frame,
1280x720, the reference generator) and the 16-stream line, with OSNet_x0_25 (seeded weights) on the device.  OccluBoost
runs configs/trackers/occluboost.yaml's parameters, BoostTrack++ configs/trackers/boosttrack.yaml's; camera-motion
estimation is off, as in every bench.py configuration.  The two trackers are timed alternately in the same process (two
rounds each, bench.py's device-resident leg with CUDA events), so the cost of OccluBoost's extra passes is a measured
difference.  Also an end-to-end leg through `OccluBoost.update(dets, img)` and parity of the first frames against the
oracle OccluBoost fed by the oracle ReID.  Prints one JSON line.

    python scripts/bench_occluboost.py [--steps 200] [--warmup 20] [--parity-frames 2]

Writes nothing into the tree (the blob goes to a temporary directory)."""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from scripts.bench_boosttrack import PARAMS as BT_PARAMS, gpu_power  # noqa: E402

OB_PARAMS = {k: v for k, v in __import__("boxmot_b200.trackers", fromlist=["x"]).OCCLUBOOST_YAML_DEFAULTS.items()
             if k not in ("use_cmc", "cmc_method", "adaptive_kf")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--parity-frames", type=int, default=2)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_occluboost.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    import boxmot_b200 as bb
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.synthetic import make_osnet_state
    from boxmot_b200.weights import export_blob

    K, Wm = args.steps, max(3, args.warmup)
    sd = make_osnet_state("osnet_x0_25", seed=0)
    blob = export_blob(sd, Path(tempfile.mkdtemp(prefix="b200ob_")) / "osnet_x0_25_synthetic.b200reid")
    bench.n_crops = lambda cfg, d: len(d)   # both embed every detection row
    lines = {}
    for S in (1, 16):
        base = bench.CONFIGS[2 if S == 1 else 5]
        runs = {"occluboost": [], "boosttrack": []}
        ps = None
        for _ in range(2):
            for kind, params in (("boosttrack", BT_PARAMS), ("occluboost", OB_PARAMS)):
                cfg = dict(base, kind=kind, params=params,
                           workload=f"{kind} + OSNet_x0_25 ReID in update(), {S} stream(s) x 256 dets/frame, 1280x720, CMC off")
                dev = bench.device_run(cfg, blob, K, Wm, None)
                ps = dev["per_stream"]
                runs[kind].append(dict(ms_per_step=dev["value_ms"] / K,
                                       association_ms_per_step=dev["prof"]["association"]["ms_per_step"],
                                       launches_per_step=dev["launches_per_step"]))
        line = {}
        for kind, r in runs.items():
            ms = float(np.mean([x["ms_per_step"] for x in r]))
            line[kind] = dict(frames_per_s=S / (ms * 1e-3), ms_per_step=ms, rounds_ms_per_step=[x["ms_per_step"] for x in r],
                              association_ms_per_step=float(np.mean([x["association_ms_per_step"] for x in r])),
                              launches_per_step=r[0]["launches_per_step"])
        line["occluboost_minus_boosttrack_ms_per_step"] = line["occluboost"]["ms_per_step"] - line["boosttrack"]["ms_per_step"]
        if S == 1:
            cfg = dict(base, kind="occluboost", params=OB_PARAMS)
            trk = bb.OccluBoost(reid_model=B200ReID(blob), use_cmc=False, cap_tracks=1024, cap_dets=256, **OB_PARAMS)
            for f in range(Wm):
                trk.update(ps[0][1][f], ps[0][0][f % cfg["ring"]])
            t0 = time.perf_counter()
            for f in range(Wm, Wm + K):
                trk.update(ps[0][1][f], ps[0][0][f % cfg["ring"]])
            e2e = 1e3 * (time.perf_counter() - t0)
            line["occluboost_e2e"] = dict(frames_per_s=K / (e2e * 1e-3), ms_per_step=e2e / K, api="OccluBoost.update(dets, img)")
            from oracle import reid as orid
            from tests.occluboost_oracle import OccluBoostOracle

            gpu = bb.OccluBoost(reid_model=B200ReID(blob), use_cmc=False, cap_tracks=1024, cap_dets=256, **OB_PARAMS)
            orc = OccluBoostOracle(reid_model=orid.OracleReID(sd), **OB_PARAMS)
            ok, n = True, 0
            for f in range(args.parity_frames):
                img = ps[0][0][f % cfg["ring"]]
                got = np.asarray(gpu.update(ps[0][1][f], img), np.float32)
                want = np.asarray(orc.update(ps[0][1][f], img), np.float32).reshape(-1, 8)
                n += len(want)
                ok = ok and got.shape == want.shape and np.array_equal(got[:, 4:], want[:, 4:])
            line["parity"] = dict(frames=args.parity_frames, rows=n, ids_conf_cls_det_ind_equal=bool(ok))
        lines[S] = line
    print(json.dumps({"metric": "OccluBoost tracker frames/sec at 256 dets/frame (device-resident leg)",
                      "value": lines[1]["occluboost"]["frames_per_s"], "unit": "frames/s", "steps": K, "warmup": Wm,
                      "device": torch.cuda.get_device_name(0), "gpu_name_power_limit_max_sm_clock": gpu_power(),
                      "one_stream": lines[1], "sixteen_streams": lines[16]}))


if __name__ == "__main__":
    main()
