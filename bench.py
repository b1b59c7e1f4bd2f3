#!/usr/bin/env python
"""bench.py -- tracker.update() frames/sec (BASELINE.json metric), GPU arm and CPU reference arm.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference] [--config 2|3|4|5] [--dump-outputs DIR]

Default workload (config.workload) = BASELINE.json configs[1]: BoT-SORT + OSNet_x0_25 ReID inside update(), one
1280x720 stream of 256 detections per frame per GPU, reference bench generator (benchmark_fps.py:60-94), YAML-default
parameters with CMC off.  `--config` selects the other BASELINE configurations:
    3  DeepOCSORT + OSNet_x1_0, 512 dets/frame out of 2048 objects in 4 cohorts (~2000 live tracks), 1920x1080
    4  StrongSORT + MobileNetV2_x1_4, 8 x 1080p streams per GPU (32 streams on 4 GPUs), 64 dets/frame each
    5  BoT-SORT + OSNet_x0_25, 16 streams x 256 dets per GPU (128 streams on 8 GPUs)
N GPUs = N independent stream groups, one process per GPU (weak scaling, no collective on the frame path; NCCL only
for the barrier and the max-over-ranks gather).

One "step" = one frame of every resident stream through the whole hot path (crop staging, ReID CNN, appearance cost,
Kalman predict/update, assignment rounds, lifecycle, output rows).
  value : stream-frames/s with frames and detections resident in HBM (ring of distinct frames larger than L2),
          timed with CUDA events on the engine's stream, max over ranks.
  e2e   : the same metric through the public API with HOST numpy buffers in PAGEABLE memory -- for one stream the
          BaseTracker-shaped `BotSort.update(dets, img)` of the reference seam -- every step copies the frame(s) +
          detections host->device and reads the result rows back (`e2e_pinned` = the same call with page-locked frames).
  roofline : SURVEY 8(d): ReID algorithmic FLOP per step (crops x FLOP/crop of the backbone) / step time, against the
          dense BF16 tensor peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet figure).
  parity : the first frames of the TIMED workload through the device path and through the oracle (outside the timed
          region): ids / det_ind / conf / cls equal, boxes within 1e-4.
  cpu_baseline : the oracle port of the reference path (numpy/scipy/torch-CPU restatement pinned to the reference by
          tests/golden) on this box's host cores, on a bounded sample of the same workload.
`--impl reference` runs that CPU arm alone and prints the same line shape.
`--dump-outputs DIR` writes the rows the timed path returned for its last step, one DIR/rows_stream<s>.npy (float32,
[rows][8]: x1 y1 x2 y2 id conf cls det_ind) per stream; inputs and ReID weights are seeded, so two builds run with the same
arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

LOCAL_RANK = int(os.environ.get("LOCAL_RANK", "0"))
RANK = int(os.environ.get("RANK", "0"))
WORLD = int(os.environ.get("WORLD_SIZE", "1"))
if WORLD > 1 and "BENCH_KEEP_VISIBLE" not in os.environ:
    vis = os.environ.get("CUDA_VISIBLE_DEVICES")
    ids = vis.split(",") if vis else [str(i) for i in range(64)]
    os.environ["CUDA_VISIBLE_DEVICES"] = ids[LOCAL_RANK % len(ids)]  # one GPU per process, device 0 inside it

import numpy as np  # noqa: E402

RING = 64  # distinct frames in the input ring of config 2: 64 x 2.76 MB = 177 MB > 50 MB of L2
BOTSORT = dict(
    track_high_thresh=0.6296854875023994, track_low_thresh=0.1014392537025336,
    new_track_thresh=0.6246494191492591, track_buffer=40, match_thresh=0.7722224024589055,
    proximity_thresh=0.6084297894561342, appearance_thresh=0.6188818853936099,
    unconfirmed_emb_scale=2.5445206391993294, second_match_thresh=0.28795081514328974,
    unconfirmed_match_thresh=0.41148010638233784, removed_stracks_buffer=329, fuse_first_associate=True,
    frame_rate=30, with_reid=True)
DEEPOCSORT = dict(det_thresh=0.5, max_age=30, min_hits=3, iou_threshold=0.3, delta_t=3, inertia=0.2, w_association_emb=0.75,
                  alpha_fixed_emb=0.95, aw_param=0.5, embedding_off=False, aw_off=False, Q_xy_scaling=0.01, Q_s_scaling=0.0001)
STRONGSORT = dict(min_conf=0.6, ema_alpha=0.9, max_cos_dist=0.4, max_iou_dist=0.7, max_age=30, n_init=3, mc_lambda=0.98, nn_budget=100)
METRIC = "tracker.update() frames/sec at 256 dets/frame"
# algorithmic GFLOP per crop (2 x MAC, convolutions + fc; SURVEY 8d)
GFLOP_PER_CROP = {"osnet_x0_25": 0.1654, "osnet_x1_0": 1.958, "mobilenetv2_x1_4": 0.764}
CONFIGS = {
    2: dict(kind="botsort", arch="osnet_x0_25", feat=512, streams=1, dets=256, hw=(720, 1280), params=BOTSORT, gen="bench",
            cap_tracks=1024, ring=RING, conf_key="track_high_thresh", strict=True,
            workload="BoT-SORT + OSNet_x0_25 ReID in update(), 1 stream x 256 dets/frame per GPU, 1280x720, CMC off"),
    3: dict(kind="deepocsort", arch="osnet_x1_0", feat=512, streams=1, dets=512, hw=(1080, 1920), params=DEEPOCSORT, gen="cohort",
            cap_tracks=2600, ring=24, conf_key="det_thresh", strict=True,
            workload="DeepOCSORT + OSNet_x1_0 ReID in update(), 512 dets/frame out of 2048 objects in 4 cohorts (~2000 live "
                     "tracks), 1920x1080, CMC off"),
    4: dict(kind="strongsort", arch="mobilenetv2_x1_4", feat=1792, streams=8, dets=64, hw=(1080, 1920), params=STRONGSORT,
            gen="bench", cap_tracks=256, ring=6, conf_key="min_conf", strict=False,
            workload="StrongSORT + MobileNetV2_x1_4 ReID in update(), 8 x 1080p streams x 64 dets/frame per GPU, CMC off"),
    5: dict(kind="botsort", arch="osnet_x0_25", feat=512, streams=16, dets=256, hw=(720, 1280), params=BOTSORT, gen="bench",
            cap_tracks=1024, ring=4, conf_key="track_high_thresh", strict=True,
            workload="BoT-SORT + OSNet_x0_25 ReID in update(), 16 streams x 256 dets/frame per GPU, 1280x720, CMC off"),
}
CLASSES = ["crop_resize_norm", "stem_conv7x7", "maxpool", "pointwise_gemm", "lightconv", "gates", "avgpool", "head",
           "association"]


# ------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------
def measured_peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return dict(hbm_gbs=float(d["hbm_gbs"]), tensor_tflops=float(d["bf16_tflops_sustained"]), source="measured")
    return dict(hbm_gbs=3350.0, tensor_tflops=989.0, source="H100 SXM data sheet (dense BF16, 700 W), not measured")


class ClockSampler:
    """nvidia-smi clocks + throttle reasons while the timed region runs."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap,power.limit")

    def __init__(self):
        self.rows = []
        self.proc = None

    def start(self):
        gpu = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", gpu], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 3 + i and r[3 + i].lower().startswith("active") for r in self.rows)]
        pl = [float(r[7]) for r in self.rows if len(r) > 7 and r[7].replace(".", "").isdigit()]
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_limit_w": max(pl) if pl else None, "reasons": reasons, "samples": len(sm)}



def make_state(arch, seed=0):
    from boxmot_b200.synthetic import make_mobilenetv2_state, make_osnet_state

    return make_mobilenetv2_state(1.4, seed=seed) if arch.startswith("mobilenetv2") else make_osnet_state(arch, seed=seed)


def make_blob(tmpdir: Path, arch: str) -> Path:
    from boxmot_b200.weights import export_blob

    return export_blob(make_state(arch), tmpdir / f"{arch}_synthetic.b200reid")


def make_inputs(cfg, stream_index: int, frames: int):
    """(images ring [ring][H][W][3] uint8, detections per frame) of one stream of the configuration."""
    from boxmot_b200.synthetic import bench_stream, cohort_stream

    if cfg["gen"] == "cohort":
        dets, _ = cohort_stream(frames=frames, hw=cfg["hw"], seed=3 + stream_index, conf_lo=0.55)
    else:
        _, dets = bench_stream(cfg["dets"], frames, hw=cfg["hw"], stream=stream_index)
    rng = np.random.default_rng(9000 + stream_index)
    imgs = rng.integers(0, 255, size=(cfg["ring"], cfg["hw"][0], cfg["hw"][1], 3), dtype=np.uint8)
    return imgs, dets


def n_crops(cfg, d):
    c = d[:, 4].astype(np.float64)
    t = cfg["params"][cfg["conf_key"]]
    return int((c > t).sum() if cfg["strict"] else (c >= t).sum())


def make_oracle(cfg, sd):
    from oracle import reid as orid

    model = orid.OracleReID(sd)
    if cfg["kind"] == "botsort":
        from oracle.trackers import BotSortOracle

        return BotSortOracle(reid_model=model, **cfg["params"])
    if cfg["kind"] == "deepocsort":
        from oracle.deepocsort import DeepOcSortOracle

        return DeepOcSortOracle(reid_model=model, **cfg["params"])
    from oracle.strongsort import StrongSortOracle

    return StrongSortOracle(reid_model=model, **cfg["params"])


# ------------------------------------------------------------------------------------------------------
# CPU arm: the oracle port of the reference path on the host cores
# ------------------------------------------------------------------------------------------------------
def cpu_arm(cfg, sample_frames: int, warm: int, budget_s: float = 25.0, stream_index: int = 0, threads: int = 0, keep_rows=False):
    """Oracle port of the reference path on the host cores, bounded by wall-clock: the host of a GPU box can be
    anything from 8 fast cores to a heavily shared 128-thread part, so the sample is 'as many frames as fit in
    `budget_s` seconds' (at least one), after a thread-count probe that is itself time-bounded.  One stream."""
    import torch

    from oracle import reid as orid

    sd = make_state(cfg["arch"])
    imgs, dets = make_inputs(cfg, stream_index, warm + sample_frames + 1)
    avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    probe_x = orid.get_crops(dets[0][:16, :4], imgs[0])
    best = (min(avail, 8), 1e30)
    t_probe = time.perf_counter()
    # `threads` > 0: one of several concurrent stream workers with a fixed share of the cores (no probe)
    for th in ([threads] if threads > 0 else sorted({min(avail, 8), min(avail, 16), min(avail, 32), avail})):
        torch.set_num_threads(th)
        t0 = time.perf_counter()
        orid.backbone_forward(sd, probe_x)
        dt = time.perf_counter() - t0
        if dt < best[1]:
            best = (th, dt)
        if time.perf_counter() - t_probe > 8.0:
            break
    cores = best[0]
    torch.set_num_threads(cores)
    trk = make_oracle(cfg, sd)
    rows = []
    t_start = time.perf_counter()
    done_warm = 0
    for f in range(warm):
        r = trk.update(dets[f], imgs[f % cfg["ring"]])
        if keep_rows:
            rows.append(np.asarray(r, np.float32).reshape(-1, 8).copy())
        done_warm += 1
        if time.perf_counter() - t_start > budget_s / 2:
            break
    t0 = time.perf_counter()
    n = 0
    for f in range(done_warm, done_warm + sample_frames):
        r = trk.update(dets[f], imgs[f % cfg["ring"]])
        if keep_rows:
            rows.append(np.asarray(r, np.float32).reshape(-1, 8).copy())
        n += 1
        if time.perf_counter() - t0 > budget_s:
            break
    dt = time.perf_counter() - t0
    out = {"value": n / dt, "unit": "frames/s", "cores": cores, "kind": "port", "frames": n, "warm": done_warm,
           "sample": f"{n} frames of one stream of the workload after {done_warm} warm-up frame(s) (time-bounded to "
                     f"~{budget_s:.0f} s), oracle port (numpy/scipy/lapjv-C + torch-CPU {cfg['arch']} fp32, {cores} of {avail} "
                     f"usable threads, fastest of a bounded thread-count probe)",
           "ms_per_frame": 1e3 * dt / n}
    if keep_rows:
        out["_rows"] = rows
    return out


def _cpu_stream_worker(job):
    cfg_id, steps, stream_index, threads = job
    return cpu_arm(CONFIGS[cfg_id], steps, 1, budget_s=40.0, stream_index=stream_index, threads=threads)


def run_reference(args):
    """The reference path on the host cores for the SAME workload as the GPU arm at this --gpus: `streams` streams per
    GPU, i.e. N x streams independent streams.  One stream: one tracker with the fastest thread count of a bounded probe.
    More: concurrent tracker processes (the reference's own replay parallelism is one process per sequence,
    engine/eval/replay.py:27-115), each with an equal share of the usable cores; value = sum of the streams' rates.
    At most 16 worker processes run (the host cores are the limit either way); the rate of the measured streams is
    scaled to the full stream count and the sample says so."""
    if RANK != 0:
        return
    cfg = CONFIGS[args.config]
    steps = max(2, min(args.steps, 12))
    n_streams = max(1, int(args.gpus)) * cfg["streams"]
    if n_streams == 1:
        base = cpu_arm(cfg, steps, 1, budget_s=40.0)
        note = "single stream on the host cores; steps bounded to keep the run short"
    else:
        import multiprocessing as mp

        avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
        workers = min(n_streams, 16)
        threads = max(1, avail // workers)
        with mp.get_context("spawn").Pool(workers) as pool:
            parts = pool.map(_cpu_stream_worker, [(args.config, steps, i, threads) for i in range(workers)])
        # all cores are busy with `workers` streams: more streams would share the same cores, the aggregate rate stays
        value = sum(p["value"] for p in parts)
        frames = min(p["frames"] for p in parts)
        base = {"value": value, "unit": "frames/s", "cores": threads * workers, "kind": "port", "frames": frames,
                "warm": min(p["warm"] for p in parts), "ms_per_frame": 1e3 / value,
                "sample": f"{workers} concurrent stream processes x {threads} threads (of {n_streams} streams in the workload; the "
                          f"host cores are saturated, the aggregate rate does not grow with more processes), "
                          f"{[p['frames'] for p in parts]} frames each after a warm-up frame (time-bounded to ~40 s), oracle port "
                          f"(numpy/scipy/lapjv-C + torch-CPU {cfg['arch']} fp32); value = sum of the per-stream rates"}
        note = f"{n_streams} independent streams on the host cores (one process per stream, {workers} at a time)"
    line = {"impl": "reference", "metric": METRIC, "value": base["value"], "unit": "frames/s", "n_gpus": args.gpus,
            "steps": base["frames"], "warmup": base["warm"], "ms_per_step": base["ms_per_frame"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": cfg["workload"], "note": note},
            "cpu_baseline": {k: base[k] for k in ("value", "unit", "cores", "kind", "sample")},
            "e2e": {"value": base["value"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


# ------------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------------
def device_run(cfg, blob, K, Wm, dist, profile=True):
    """value (device-resident inputs, CUDA events) + the per-class profile of one configuration on this rank's GPU."""
    import torch

    import boxmot_b200 as bb
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    S, CD, (H, Wd) = cfg["streams"], cfg["dets"], cfg["hw"]
    ring = cfg["ring"]
    per_stream = [make_inputs(cfg, RANK * S + s, Wm + K + 8) for s in range(S)]
    crops = float(np.mean([sum(n_crops(cfg, per_stream[s][1][f]) for s in range(S)) for f in range(Wm, Wm + K)]))

    def new_tracker():
        return bb.MultiStreamTracker(cfg["kind"], n_streams=S, cap_tracks=cfg["cap_tracks"], cap_dets=CD, feat_dim=cfg["feat"],
                                     reid_blob=str(blob), **cfg["params"])

    trk = new_tracker()
    # [ring][S][H][W][3] u8; frame f of every stream uses detections f of that stream and ring slot f % ring
    d_imgs = torch.from_numpy(np.stack([p[0] for p in per_stream], 1)).cuda()
    nf = Wm + K + 8
    dd = np.zeros((nf, S, CD, 6), np.float32)
    rows_np = np.zeros((nf, S), np.int32)
    for s in range(S):
        for f in range(nf):
            d = per_stream[s][1][f][:CD]
            dd[f, s, : len(d)] = d
            rows_np[f, s] = len(d)
    d_dets = torch.from_numpy(dd).cuda()
    torch.cuda.synchronize()

    def dev_step(f, sync=0):
        rows = (ctypes.c_int * S)(*[int(x) for x in rows_np[f]])
        ok = lib.boxmot_b200_tracker_update_device(trk.handle, d_dets[f].data_ptr(), rows, None,
                                                   d_imgs[f % ring].data_ptr(), H, Wd, sync)
        if not ok:
            raise RuntimeError(_lib.last_error(lib))

    for f in range(Wm):
        dev_step(f, 1)
    launches_per_step = trk.last_launches()
    torch.cuda.synchronize()
    if dist:
        dist.barrier()
    clocks = ClockSampler()
    clocks.start()
    lib.boxmot_b200_tracker_mark(trk.handle, 0)
    for f in range(Wm, Wm + K):
        dev_step(f, 0)
    lib.boxmot_b200_tracker_mark(trk.handle, 1)
    ms = ctypes.c_double(0)
    if not lib.boxmot_b200_tracker_elapsed_ms(trk.handle, ctypes.byref(ms)):
        raise RuntimeError(_lib.last_error(lib))
    torch.cuda.synchronize()
    last_rows = [np.asarray(r, np.float32).reshape(-1, 8) for r in trk.fetch()]   # surfaces device-side errors
    value_ms = ms.value
    prof, assoc_phases = None, None
    if profile:
        # events around every launch, serialised on one stream (no slice concurrency, no frame pipeline)
        phase = (ctypes.c_longlong * 16)()
        lib.boxmot_b200_tracker_phase_clocks(trk.handle, 0, phase, 1)
        lib.boxmot_b200_tracker_profile(trk.handle, 1)
        P = min(16, K)
        for f in range(Wm + K - P, Wm + K):
            dev_step(f, 1)
        cls_ms = (ctypes.c_double * 9)()
        cls_n = (ctypes.c_int * 9)()
        lib.boxmot_b200_tracker_profile_read(trk.handle, cls_ms, cls_n)
        lib.boxmot_b200_tracker_profile(trk.handle, 0)
        lib.boxmot_b200_tracker_phase_clocks(trk.handle, 0, phase, 1)
        phase_names = ["split+predict", "cost1", "assign1", "update1", "round2", "round3", "births+lists", "dups+output"]
        assoc_phases = {n: phase[i] / P for i, n in enumerate(phase_names)}
        prof = {CLASSES[i]: {"ms_per_step": cls_ms[i] / P, "launches_per_step": cls_n[i] / P} for i in range(9)}
    clock_info = clocks.stop()
    trk.close()
    del d_imgs, d_dets
    torch.cuda.empty_cache()
    return dict(value_ms=value_ms, crops=crops, launches_per_step=launches_per_step, prof=prof, assoc_phases=assoc_phases,
                clocks=clock_info, per_stream=per_stream, new_tracker=new_tracker, last_rows=last_rows)


def e2e_run(cfg, blob, per_stream, K, Wm, dist, pinned):
    """stream-frames/s through the public API with host numpy buffers; one synchronous call per frame."""
    import torch

    import boxmot_b200 as bb
    from boxmot_b200.reid import B200ReID

    S, ring = cfg["streams"], cfg["ring"]
    imgs = [p[0] for p in per_stream]
    if pinned:
        keep = [torch.from_numpy(im).pin_memory() for im in imgs]
        imgs = [k.numpy() for k in keep]
    if S == 1:
        # the BaseTracker-shaped seam of the reference: tracker.update(dets, img) -> (M, 8) rows
        cls = {"botsort": bb.BotSort, "deepocsort": bb.DeepOcSort, "strongsort": bb.StrongSort}[cfg["kind"]]
        trk = cls(reid_model=B200ReID(blob), cap_tracks=cfg["cap_tracks"], cap_dets=cfg["dets"], **cfg["params"])
        step = lambda f: trk.update(per_stream[0][1][f], imgs[0][f % ring])   # noqa: E731
        api = f"{cls.__name__}.update(dets, img)"
    else:
        trk = bb.MultiStreamTracker(cfg["kind"], n_streams=S, cap_tracks=cfg["cap_tracks"], cap_dets=cfg["dets"],
                                    feat_dim=cfg["feat"], reid_blob=str(blob), **cfg["params"])
        step = lambda f: trk.update([per_stream[s][1][f] for s in range(S)], [imgs[s][f % ring] for s in range(S)])   # noqa: E731
        api = "MultiStreamTracker.update(dets per stream, images per stream)"
    for f in range(Wm):
        step(f)
    torch.cuda.synchronize()
    if dist:
        dist.barrier()
    t0 = time.perf_counter()
    last = None
    for f in range(Wm, Wm + K):
        last = step(f)
    ms = 1e3 * (time.perf_counter() - t0)
    n_out = int(len(last)) if S == 1 else int(sum(len(x) for x in last))
    if hasattr(trk, "close"):
        trk.close()
    return ms, n_out, api


def parity_check(cfg, blob, oracle_rows, per_stream):
    """The first frames of the timed workload (stream 0 of this rank) through the device path, against the oracle rows the
    cpu_baseline leg produced for exactly those frames."""
    import boxmot_b200 as bb
    from boxmot_b200.reid import B200ReID

    cls = {"botsort": bb.BotSort, "deepocsort": bb.DeepOcSort, "strongsort": bb.StrongSort}[cfg["kind"]]
    trk = cls(reid_model=B200ReID(blob), cap_tracks=cfg["cap_tracks"], cap_dets=cfg["dets"], **cfg["params"])
    ids_equal, boxes_ok, n_rows = True, True, 0
    for f, want in enumerate(oracle_rows):
        got = np.asarray(trk.update(per_stream[0][1][f], per_stream[0][0][f % cfg["ring"]]), np.float32).reshape(-1, 8)
        n_rows += len(want)
        if got.shape != want.shape or not np.array_equal(got[:, 4:], want[:, 4:]):
            ids_equal = False
            break
        if len(want) and not np.allclose(got[:, :4], want[:, :4], rtol=1e-4, atol=1e-3):
            boxes_ok = False
    return {"frames": len(oracle_rows), "rows": n_rows, "ids_equal": bool(ids_equal), "boxes_within_1e-4": bool(boxes_ok and ids_equal),
            "what": "ids, det_ind, conf, cls of every output row of the first frames of the timed stream, device vs oracle"}


def dump_outputs(out_dir, rows):
    """Rows of the last timed step, one float32 file per stream (a few hundred rows each: far below 64 MB)."""
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    for s, r in enumerate(rows):
        np.save(d / f"rows_stream{RANK * len(rows) + s}.npy", np.asarray(r, np.float32))


def run_b200(args):
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    dist = None
    if WORLD > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=torch.device("cuda:0"))
    cfg = dict(CONFIGS[args.config], id=args.config)
    K, Wm = args.steps, max(3, args.warmup)
    tmp = Path(tempfile.mkdtemp(prefix="b200bench_"))
    blob = make_blob(tmp, cfg["arch"])
    S = cfg["streams"]
    H, Wd = cfg["hw"]
    img_bytes = H * Wd * 3

    dev = device_run(cfg, blob, K, Wm, dist)
    value_ms, crops, prof = dev["value_ms"], dev["crops"], dev["prof"]
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, dev["last_rows"])
    e2e_ms, n_out, api = e2e_run(cfg, blob, dev["per_stream"], K, Wm, dist, pinned=False)
    e2e_pin_ms, _, _ = e2e_run(cfg, blob, dev["per_stream"], K, Wm, dist, pinned=True)

    extra5 = None
    if args.config == 2 and not args.no_extra:
        # BASELINE config 5 shape on the same GPUs (16 streams x 256 dets per GPU), same steps: the scaling run then carries
        # the 128-stream figure at N = 8 beside the one-stream-per-GPU headline
        c5 = dict(CONFIGS[5], id=5)
        d5 = device_run(c5, blob, K, Wm, dist, profile=False)
        extra5 = (d5["value_ms"], d5["crops"])

    from boxmot_b200 import sharding

    red = [value_ms, e2e_ms, e2e_pin_ms] + ([extra5[0]] if extra5 else [])
    red = sharding.reduce_max(red, dist, device="cuda")  # slowest rank defines the job
    value_ms, e2e_ms, e2e_pin_ms = red[0], red[1], red[2]
    frames_per_rank = sharding.gather_counts(S * K, dist, device="cuda")
    if RANK != 0:
        if dist:
            dist.barrier()
            dist.destroy_process_group()
        return
    peaks = measured_peaks()
    total_frames = sum(frames_per_rank)
    fps = total_frames / (value_ms * 1e-3)
    e2e_fps = total_frames / (e2e_ms * 1e-3)
    step_s = value_ms * 1e-3 / K
    gflop_step = crops * GFLOP_PER_CROP[cfg["arch"]]                  # per rank per step
    achieved = gflop_step / step_s / 1e3                              # TFLOP/s per GPU
    reid_ms = sum(prof[c]["ms_per_step"] for c in CLASSES if c != "association")
    dom = max((c for c in CLASSES if c != "association"), key=lambda c: prof[c]["ms_per_step"])
    tc_path = cfg["arch"] == "osnet_x0_25"
    line = {
        "metric": METRIC, "value": fps, "unit": "frames/s", "n_gpus": WORLD, "steps": K, "warmup": Wm,
        "ms_per_step": value_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "bf16x3" if tc_path else "f32", "data": "synthetic",
        "config": {"workload": cfg["workload"], "baseline_config": args.config, "streams_per_gpu": S, "dets_per_frame": cfg["dets"],
                   "crops_per_step_per_gpu": crops,
                   "reid": f"{cfg['arch']} random-init (seed 0); " + (
                       "tensor-core path: wgmma on split-BF16 operands (hi*hi + lo*hi + hi*lo, FP32 accumulate), depthwise / "
                       "pooling / gates in float32" if tc_path else "float32 CUDA-core kernels"),
                   "l2": f"input ring of {cfg['ring']} distinct frames per stream ({cfg['ring'] * S * img_bytes / 1e6:.0f} MB) and a "
                         f"per-chunk activation workspace larger than L2; no explicit flush",
                   "parallelism": f"streams x{WORLD * S} ({S} per GPU)",
                   "value_path": "update_device, device-resident inputs, no per-frame sync: ReID of frame f+1 overlaps "
                                 "the association of frame f on two CUDA streams",
                   "e2e_path": f"{api} per frame with PAGEABLE numpy frames: frame H2D (staged through a pinned buffer) + dets "
                               "H2D, full sync, rows D2H"},
        "e2e": {"value": e2e_fps, "unit": "frames/s", "ms_per_step": e2e_ms / K,
                "h2d_bytes_per_step": S * (img_bytes + cfg["dets"] * 6 * 4 + 4),
                "d2h_bytes_per_step": S * (cfg["dets"] * 8 * 4 + 16 * 4), "rows_last_frame": n_out, "api": api,
                "host_memory": "pageable"},
        "e2e_pinned": {"value": total_frames / (e2e_pin_ms * 1e-3), "unit": "frames/s", "ms_per_step": e2e_pin_ms / K,
                       "host_memory": "page-locked frames (copied straight from the caller's buffer)"},
        "device": torch.cuda.get_device_name(0),
        "gpu_launches": dev["launches_per_step"] * K,
        "launches_per_step": dev["launches_per_step"],
        "clocks": dev["clocks"],
        # SURVEY 8(d): achieved = crops/s x FLOP/crop of the backbone, per GPU, over the measured step time
        "roofline": {"kernel": "ReID backbone (all conv / fc kernels of a step)", "bound": "tensor", "achieved": achieved,
                     "peak": peaks["tensor_tflops"], "unit": "TFLOP/s", "frac": achieved / peaks["tensor_tflops"],
                     "peak_source": peaks["source"],
                     "algorithmic_gflop_per_step": gflop_step, "gflop_per_crop": GFLOP_PER_CROP[cfg["arch"]],
                     "step_ms": value_ms / K,
                     "note": "the tensor-core path issues 3 BF16 products per algorithmic MAC (split operands), so 1/3 of the "
                             "tensor work is algorithmic",
                     "serialised_reid_ms_per_step": reid_ms,
                     "frac_serialised": gflop_step / (reid_ms * 1e-3) / 1e3 / peaks["tensor_tflops"],
                     "dominant_class": dom, "dominant_class_ms": prof[dom]["ms_per_step"]},
        "kernel_classes": prof,
        "association_phase_sm_clocks_per_step": dev["assoc_phases"],
    }
    if extra5:
        fps5 = WORLD * CONFIGS[5]["streams"] * K / (red[3] * 1e-3)
        line["config5"] = {"workload": CONFIGS[5]["workload"], "value": fps5, "unit": "frames/s", "streams": WORLD * CONFIGS[5]["streams"],
                           "ms_per_step": red[3] / K, "steps": K,
                           "reid_tflops_per_gpu": extra5[1] * GFLOP_PER_CROP["osnet_x0_25"] / (red[3] * 1e-3 / K) / 1e3,
                           "frac_of_tensor_peak": extra5[1] * GFLOP_PER_CROP["osnet_x0_25"] / (red[3] * 1e-3 / K) / 1e3 / peaks["tensor_tflops"]}
    if WORLD == 1 and not args.skip_cpu:
        cb = cpu_arm(cfg, args.cpu_frames, 1, keep_rows=True)
        rows = cb.pop("_rows")
        line["cpu_baseline"] = cb
        line["speedup_e2e_vs_cpu"] = e2e_fps / (S * cb["value"])
        line["parity"] = parity_check(cfg, blob, rows, dev["per_stream"])
    print(json.dumps(line))
    if dist:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200,
                    help="timed steps of the GPU arm (headline, e2e and config-5 legs); the CPU reference arm (--impl reference) "
                         "times at most 12 frames within ~40 s, the cpu_baseline leg --cpu-frames within ~25 s")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", type=int, default=2, choices=[2, 3, 4, 5], help="BASELINE.json configuration (default: the headline)")
    ap.add_argument("--cpu-frames", type=int, default=8)
    ap.add_argument("--skip-cpu", action="store_true", help="kernel A/B experiments only: omit the cpu_baseline / parity legs")
    ap.add_argument("--no-extra", action="store_true", help="omit the short config-5 (16 streams per GPU) measurement")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the rows of the last timed step as DIR/rows_stream<s>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_b200(args)


if __name__ == "__main__":
    main()
